"""Longest dependency path of the captured iteration graph.

Inputs:
  graph.dot     MAML_B200_GRAPH_DOT=<file> python scripts/trace_timeline.py            (cudaGraphDebugDotPrint)
  serial trace  MAML_B200_ONE_STREAM=1 python scripts/trace_timeline.py --full > <file>  (true kernel durations: one stream)
Kernel nodes of the graph (creation order) and trace entries (launch order) are the same sequence, so node i gets the
serial "time to next start" of entry i as its cost; the longest path through the DAG is what an ideal machine with
unlimited SMs would need.  Prints the path's composition per kernel and the slack of everything else.

    python scripts/critical_path.py gpurun_out/graph.dot gpurun_out/trace_serial.txt
"""
import collections
import re
import sys


def main():
    import json, os
    ids = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "trace_kernel_ids.json")))
    global KNOWN
    KNOWN = sorted(ids, key=len, reverse=True)
    dot, trace = sys.argv[1], sys.argv[2]
    txt = open(dot).read()
    nodes = {}
    for m in re.finditer(r'"(graph_\d+_node_(\d+))"\[[^\]]*?label="(\d+)\n([^"]*)"\]', txt, re.S):
        name, idx, body = m.group(1), int(m.group(2)), m.group(4)
        first = body.split("\n")[0]
        is_kernel = "<<<" in body.replace("\\<", "<")
        km = None
        for cand in KNOWN:
            if cand in first:
                km = re.match("(.*)", cand)
                break
        grid = re.search(r"\\<\\<\\<\\\{([^\\]*)\\\}", body)
        nodes[name] = dict(idx=idx, kernel=is_kernel, name=km.group(1) if km else first[:24],
                           grid=grid.group(1) if grid else "")
    edges = re.findall(r'"(graph_\d+_node_\d+)" -> "(graph_\d+_node_\d+)"', txt)
    # serial durations
    durs = []
    for line in open(trace):
        m = re.match(r"\s*([\d.]+) us\s+(\S+)\s+\+(-?[\d.]+)", line)
        if m:
            durs.append((m.group(2), float(m.group(3))))
    # fold conv_tc:end gaps into the conv entry before them
    ents = []
    for nm, d in durs:
        if nm.endswith(":end"):
            ents[-1] = (ents[-1][0], ents[-1][1] + d)
        else:
            ents.append((nm, d))
    knodes = sorted([n for n in nodes.values() if n["kernel"]], key=lambda n: n["idx"])
    print("graph: %d nodes (%d kernels), %d edges; trace: %d kernel entries" % (len(nodes), len(knodes), len(edges), len(ents)))
    while len(ents) > len(knodes) and ents[-1][0] in ("adam", "running_update"):     # separate C-ABI calls, not in the graph
        ents.pop()
    assert len(knodes) == len(ents), "graph / trace kernel counts differ"
    for n, (nm, d) in zip(knodes, ents):
        assert nm.split("_")[0][:4] in n["name"], (nm, n["name"])
        n["cost"] = d
        n["tname"] = nm
    for n in nodes.values():
        n.setdefault("cost", 1.0)       # memset / event nodes
        n.setdefault("tname", n["name"])
    succ = collections.defaultdict(list)
    pred = collections.defaultdict(list)
    for a, b in edges:
        succ[a].append(b)
        pred[b].append(a)
    order = sorted(nodes, key=lambda k: nodes[k]["idx"])      # creation order is a topological order
    est, best = {}, {}
    for k in order:
        s = 0.0
        bp = None
        for p in pred[k]:
            if est[p] + nodes[p]["cost"] > s:
                s, bp = est[p] + nodes[p]["cost"], p
        est[k], best[k] = s, bp
    end = max(order, key=lambda k: est[k] + nodes[k]["cost"])
    total = est[end] + nodes[end]["cost"]
    path = []
    k = end
    while k is not None:
        path.append(k)
        k = best[k]
    path.reverse()
    serial = sum(n["cost"] for n in nodes.values())
    print("serial sum %.0f us; longest path %.0f us over %d nodes" % (serial, total, len(path)))
    agg = collections.OrderedDict()
    for k in path:
        n = nodes[k]
        key = n["tname"] + " {" + n["grid"] + "}"
        c, s = agg.get(key, (0, 0.0))
        agg[key] = (c + 1, s + n["cost"])
    print("critical path by kernel {grid}:")
    for key, (c, s) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print("  %-40s n=%3d  %7.1f us  (%4.1f%%)  mean %.1f" % (key, c, s, 100 * s / total, s / c))
    # latest start times -> slack
    lst = {}
    for k in reversed(order):
        t = total
        for q in succ[k]:
            t = min(t, lst[q])
        lst[k] = t - nodes[k]["cost"]
    off = collections.OrderedDict()
    onpath = set(path)
    for k in order:
        if k in onpath or not nodes[k]["kernel"]:
            continue
        n = nodes[k]
        key = n["tname"]
        c, s, sl = off.get(key, (0, 0.0, 1e9))
        off[key] = (c + 1, s + n["cost"], min(sl, lst[k] - est[k]))
    print("off the path (count, summed cost, min slack):")
    for key, (c, s, sl) in sorted(off.items(), key=lambda kv: -kv[1][1]):
        print("  %-22s n=%3d  %7.1f us   min slack %.1f us" % (key, c, s, sl))
    if "--path" in sys.argv:
        for k in path:
            n = nodes[k]
            print("   %8.1f  %-22s {%s}  %.1f" % (est[k], n["tname"], n["grid"], n["cost"]))


if __name__ == "__main__":
    main()
