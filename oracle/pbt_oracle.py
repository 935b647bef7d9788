"""Plain-Python restatement of one ``pbt`` suggestion call (test-only; the service is kubeflow_b200/suggestion/pbt_service.py,
whose docstring states the rules, the [RECALL] list and this engine's choices).

Input: the known trials as dicts {name, generation, parent, predecessor, params, objective, condition} (condition one of
"running", "succeeded", "failed"; "succeeded" without an objective counts as failed), the search space as dicts
{name, type, min, max, list}, the goal ("MINIMIZE" / "MAXIMIZE"), the settings {n_population, truncation_threshold,
resample_probability}, anything with a ``random()`` method returning uniforms in [0, 1) (a numpy.random.Generator, or a
scripted list in hand-worked tests), the request size k and the experiment name.
Output: per issued trial {trial_name, params, labels, copy_from} (copy_from: the parent whose checkpoint directory the trial's
directory copies, or None for an empty one).
"""
from __future__ import annotations

import math

LABEL = "pbt.suggestion.katib.kubeflow.org/"
ALPHABET = "abcdefghijklmnopqrstuvwxyz0123456789"


def prior_draw(spec, u):
    if spec["type"] == "double":
        return repr(float(spec["min"]) + u * (float(spec["max"]) - float(spec["min"])))
    if spec["type"] == "int":
        lo, hi = int(spec["min"]), int(spec["max"])
        return str(min(lo + math.floor(u * (hi - lo + 1)), hi))
    n = len(spec["list"])
    return spec["list"][min(math.floor(u * n), n - 1)]


def perturb(spec, value, u):
    """Multiply by 0.8 (u < 1/2) or 1.2; integers: round half up, step by one in the factor's direction when rounding left the
    value where it was; clip.  Lists: the previous (u < 1/2) or the next entry, clamped at the ends."""
    down = u < 0.5
    if spec["type"] == "double":
        x = float(value) * (0.8 if down else 1.2)
        return repr(min(max(x, float(spec["min"])), float(spec["max"])))
    if spec["type"] == "int":
        v = int(value)
        x = math.floor(v * (0.8 if down else 1.2) + 0.5)
        if x == v:
            grows = (v > 0 and not down) or (v < 0 and down) or (v == 0 and not down)
            x = v + 1 if grows else v - 1
        return str(min(max(x, int(spec["min"])), int(spec["max"])))
    lst = spec["list"]
    i = lst.index(value)
    j = i - 1 if down else i + 1
    return lst[min(max(j, 0), len(lst) - 1)]


def truncation_count(threshold, n_members):
    return math.floor(threshold * n_members + 1e-9)


def rank_members(members, goal):
    """Best first; ties: lower generation, then name."""
    sign = 1.0 if goal == "MINIMIZE" else -1.0
    return sorted(members, key=lambda t: (sign * t["objective"], t["generation"], t["name"]))


def name_prefix(experiment):
    s = "".join(c if ("a" <= c <= "z" or "0" <= c <= "9" or c == "-") else "-" for c in experiment.lower())
    return s[:54].strip("-")


def new_name(experiment, rng, taken):
    while True:
        tail = "".join(ALPHABET[min(math.floor(rng.random() * 36), 35)] for _ in range(8))
        name = name_prefix(experiment) + "-" + tail if name_prefix(experiment) else tail
        if name not in taken:
            return name


def step(trials, space, goal, settings, rng, k, experiment):
    def finished_ok(t):
        return t["condition"] == "succeeded" and t["objective"] is not None

    def ended(t):
        return t["condition"] in ("succeeded", "failed") and not finished_ok(t)

    known = {t["name"]: t for t in trials}
    has_successor = {t["predecessor"] for t in trials if t["predecessor"] is not None}
    slots_now = [t for t in trials if t["name"] not in has_successor]

    members = []
    for t in slots_now:
        if finished_ok(t):
            members.append(t)
        elif t["condition"] == "running" and t["parent"] is not None:
            before = known.get(t["predecessor"])
            if before is not None and finished_ok(before):
                members.append(before)
    ranked = rank_members(members, goal)
    cut = truncation_count(settings["truncation_threshold"], len(ranked))
    top = ranked[:cut]
    bottom = {t["name"] for t in ranked[len(ranked) - cut:]} if cut else set()

    started = len([t for t in trials if t["predecessor"] is None])
    queue = [None] * max(settings["n_population"] - started, 0)
    queue += sorted([t for t in slots_now if t["condition"] != "running"], key=lambda t: (t["generation"], t["name"]))

    out, taken = [], set(known)
    for slot in queue[:k]:
        if slot is None or ended(slot):
            parent = None
            params = {s["name"]: prior_draw(s, rng.random()) for s in space}
        elif slot["name"] not in bottom:
            parent = slot
            params = {s["name"]: slot["params"][s["name"]] for s in space}
        else:
            parent = top[min(math.floor(rng.random() * len(top)), len(top) - 1)]
            params = {}
            for s in space:
                p = settings.get("resample_probability")
                if p is not None and rng.random() < p:
                    params[s["name"]] = prior_draw(s, rng.random())
                else:
                    params[s["name"]] = perturb(s, parent["params"][s["name"]], rng.random())
        name = new_name(experiment, rng, taken)
        taken.add(name)
        labels = {LABEL + "generation": str(parent["generation"] + 1 if parent else 0)}
        if parent:
            labels[LABEL + "parent"] = parent["name"]
        if slot:
            labels[LABEL + "predecessor"] = slot["name"]
        out.append({"trial_name": name, "params": params, "labels": labels, "copy_from": parent["name"] if parent else None})
    return out
