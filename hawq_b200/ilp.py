"""Mixed-precision bit allocation (SURVEY.md 8(f) rank 4; reference: ILP.ipynb cells 5-14 / 18-27).

HAWQ-V3 chooses 4 or 8 bits per layer by an integer linear program: minimise the second-order sensitivity
``sum_i x_i * trace_i * (||dW_i||^2_8bit - ||dW_i||^2_4bit)`` (x_i = 1 for 8 bit; every term is negative, 8 bit is always
preferred) under ONE budget — model size, BOPS or measured latency — with the residual-branch convolution of a resize unit tied
to the unit's first convolution (they read the same activation).  With a single budget this is a 0/1 knapsack; the reference hands
it to GLPK through pulp, neither of which is available here, so :func:`solve` is a small exact branch-and-bound (fractional-knapsack
bound).  ``layer_order`` / ``tie_pairs`` give the reference's variable numbering so results map onto ``bit_config.py`` entries, and
:func:`latency_table_from_detail` turns per-launch timings of this engine (``bench.py --detail``) into the ``latency_int4`` /
``latency_int8`` arrays the notebook expects, i.e. this engine's replacement of the reference's T4 table (ILP.ipynb cells 4 / 17).
"""
import numpy as np


def layer_order(arch):
    """Module names in the notebook's variable order (first convolution and classifier excluded, ILP.ipynb cell 4 comment)."""
    units, bottleneck = {"resnet18": ([2, 2, 2, 2], False), "resnet50": ([3, 4, 6, 3], True), "resnet101": ([3, 4, 23, 3], True)}[arch]
    names = []
    for s, n in enumerate(units):
        for u in range(n):
            base = "stage%d.unit%d." % (s + 1, u + 1)
            for k in range(3 if bottleneck else 2):
                names.append(base + "quant_convbn%d" % (k + 1))
            if u == 0 and (bottleneck or s > 0):
                names.append(base + "quant_identity_convbn")
    return names


def tie_pairs(arch):
    """(i, j) variable pairs forced equal: a resize unit's first convolution and its identity convolution."""
    names = layer_order(arch)
    idx = {n: i for i, n in enumerate(names)}
    return [(idx[n.replace("quant_identity_convbn", "quant_convbn1")], i) for i, n in enumerate(names) if n.endswith("quant_identity_convbn")]


def budget(cost4, cost8, fraction):
    """The notebook's limit: all-4-bit cost + fraction * (all-8-bit cost - all-4-bit cost) (ILP.ipynb cell 5)."""
    c4, c8 = float(np.sum(cost4)), float(np.sum(cost8))
    return c4 + (c8 - c4) * fraction


def solve(sensitivity, cost4, cost8, limit, ties=()):
    """Exact solution of  min sum_i x_i * sensitivity_i  s.t.  sum_i (cost4_i + x_i * (cost8_i - cost4_i)) <= limit,
    x_i in {0, 1}, x_a == x_b for (a, b) in ties.  Returns bits per layer (4 / 8) as a list."""
    s = np.asarray(sensitivity, dtype=np.float64)
    c4 = np.asarray(cost4, dtype=np.float64)
    c8 = np.asarray(cost8, dtype=np.float64)
    n = len(s)
    group = list(range(n))
    for a, b in ties:                                  # union by relabelling (tiny n)
        ga, gb = group[a], group[b]
        group = [ga if g == gb else g for g in group]
    reps = sorted(set(group))
    value = np.array([-s[[i for i in range(n) if group[i] == g]].sum() for g in reps])            # gain of going to 8 bit
    weight = np.array([(c8 - c4)[[i for i in range(n) if group[i] == g]].sum() for g in reps])     # cost of going to 8 bit
    cap = float(limit) - float(c4.sum())
    take = np.zeros(len(reps), dtype=bool)
    free = (weight <= 0) & (value >= 0)                # 8 bit is no more expensive than 4 bit (e.g. this engine's 4-bit layers, which run on int8 MMA): take
    if cap - float(weight[free].sum()) < -1e-9:
        raise ValueError("infeasible: the budget is below the cheapest assignment")
    order = [i for i in np.argsort(-(value / np.maximum(weight, 1e-300))) if not free[i] and value[i] > 0]
    best = {"val": -1.0, "set": None}

    def bound(k, val, room):
        for i in order[k:]:
            if weight[i] <= room:
                room -= weight[i]; val += value[i]
            else:
                return val + value[i] * room / weight[i]
        return val

    def rec(k, val, room, chosen):
        if val > best["val"]:
            best["val"], best["set"] = val, list(chosen)
        if k == len(order) or bound(k, val, room) <= best["val"] + 1e-15:
            return
        i = order[k]
        if weight[i] <= room + 1e-12:
            chosen.append(i)
            rec(k + 1, val + value[i], room - weight[i], chosen)
            chosen.pop()
        rec(k + 1, val, room, chosen)

    import sys
    old = sys.getrecursionlimit()
    sys.setrecursionlimit(max(old, 10000))
    try:
        rec(0, 0.0, cap - float(weight[free].sum()), [])
    finally:
        sys.setrecursionlimit(old)
    take[free] = True
    for i in best["set"] or []:
        take[i] = True
    gbit = {g: (8 if take[j] else 4) for j, g in enumerate(reps)}
    return [gbit[group[i]] for i in range(n)]


def allocate(data, constraint, fraction, arch):
    """The notebook's three problems on one data dictionary (keys as in ILP.ipynb cells 4 / 17)."""
    sens = np.asarray(data["Hutchinson_trace"]) * (np.asarray(data["delta_weights_8bit_square"]) - np.asarray(data["delta_weights_4bit_square"]))
    if constraint == "modelsize":                      # 0.5 * x * parameters with x in {1, 2}  (cell 8)
        c4, c8 = 0.5 * np.asarray(data["parameters"]), 1.0 * np.asarray(data["parameters"])
    elif constraint == "bops":                         # bops / 8 / 8 and bops / 4 / 4  (cell 5)
        c4, c8 = np.asarray(data["bops"]) / 64.0, np.asarray(data["bops"]) / 16.0
    elif constraint == "latency":
        c4, c8 = np.asarray(data["latency_int4"]), np.asarray(data["latency_int8"])
    else:
        raise ValueError("constraint must be modelsize / bops / latency")
    bits = solve(sens, c4, c8, budget(c4, c8, fraction), tie_pairs(arch))
    return dict(zip(layer_order(arch), bits))


def latency_table_from_detail(detail4, detail8, arch, parameters):
    """(latency_int4, latency_int8) in ms, in the notebook's variable order, from two ``bench.py --detail`` files of this engine
    (uniform4 and uniform8 runs of ``arch``).  The launches of a forward are: stem, pool, then per unit conv1, conv2 and the last
    convolution — for resize units either one fused launch (``hawq_conv2d_dual``: last conv + identity conv) or the identity
    convolution followed by the last one; fused launches are split in proportion to the two layers' parameter counts (both are
    1x1 convolutions on the same output grid, so MACs are proportional to parameters)."""
    names = layer_order(arch)
    idx = {n: i for i, n in enumerate(names)}
    bottleneck = any(n.endswith("quant_convbn3") for n in names)
    last = "quant_convbn3" if bottleneck else "quant_convbn2"
    tables = []
    for det in (detail4, detail8):
        launches = iter([l for l in det["layers"] if l["kernel"].startswith(("hawq_conv2d", "conv"))])
        lat = np.zeros(len(names))
        units = sorted({n.rsplit(".", 1)[0] for n in names}, key=lambda u: [int(t) for t in u.replace("stage", "").replace("unit", "").split(".")])
        for u in units:
            resize = (u + ".quant_identity_convbn") in idx
            for k in range(1, 3 if bottleneck else 2):
                lat[idx["%s.quant_convbn%d" % (u, k)]] = next(launches)["ms"]
            l = next(launches)
            if not resize:
                lat[idx[u + "." + last]] = l["ms"]
            elif l["kernel"] in ("hawq_conv2d_dual", "conv_tc_dual", "conv_dual"):
                a, b = idx[u + "." + last], idx[u + ".quant_identity_convbn"]
                w = parameters[a] / (parameters[a] + parameters[b])
                lat[a], lat[b] = l["ms"] * w, l["ms"] * (1 - w)
            else:                                      # identity convolution launched on its own, then the last convolution
                lat[idx[u + ".quant_identity_convbn"]] = l["ms"]
                lat[idx[u + "." + last]] = next(launches)["ms"]
        if next(launches, None) is not None:
            raise ValueError("more convolution launches than layers: not a %s detail file" % arch)
        tables.append(lat)
    return tables[0], tables[1]
