#!/usr/bin/env python3
"""Extract the reference's known-answer tables for the requirement algebra into tests/golden/requirement_kats.json.

Sources, in a checkout of the reference given as the first argument:
  pkg/scheduling/requirement_test.go    Intersection tables (with / without minValues), Has, Operator, Len
  pkg/scheduling/requirements_test.go   Compatible matrices (AllowUndefinedWellKnownLabels and strict)

The Go sources are parsed textually: `name := NewRequirement[WithFlexibility](key, op, [minValues,] values...)`
definitions build a symbol table; `Entry(nil, a, b, expected)` rows and `Expect(a.Compatible(b[, opt])).To[Not](Succeed())`
lines are emitted as operator-form vectors.  Run once here; the JSON is committed.
"""
import json
import re
import sys

REF = sys.argv[1]
OPS = {"NodeSelectorOpIn": "In", "NodeSelectorOpNotIn": "NotIn", "NodeSelectorOpExists": "Exists",
       "NodeSelectorOpDoesNotExist": "DoesNotExist", "NodeSelectorOpGt": "Gt", "NodeSelectorOpLt": "Lt",
       "NodeSelectorOpGte": "Gte", "NodeSelectorOpLte": "Lte"}


def strings(s):
    return re.findall(r'"([^"]*)"', s)


def parse_defs(src, wrapped=False):
    sym = {}
    pat = re.compile(r"(\w+)\s*:=\s*(?:NewRequirements\()?NewRequirement(WithFlexibility)?\(([^\n]*)\)\s*$", re.M)
    for m in pat.finditer(src):
        name, flex, args = m.group(1), m.group(2), m.group(3)
        op = OPS[re.search(r"NodeSelectorOp\w+", args).group(0)]
        mv = None
        rest = args[args.index("NodeSelectorOp"):]
        if flex:
            mm = re.search(r"lo\.ToPtr\((\d+)\)", rest)
            mv = int(mm.group(1)) if mm else None
        vals = strings(rest)
        if "strconv.Itoa(math.MaxInt)" in rest:
            vals = [str(2**63 - 1)]
        sym[name] = {"op": op, "values": vals, "min_values": mv}
    return sym


def parse_literal(expr, sym):
    """&Requirement{Key: "key", complement: true, values: sets.New("A"), gte: greaterThan1.gte, MinValues: lo.ToPtr(1)}"""
    out = {"complement": "complement: true" in expr, "values": [], "gte": None, "lte": None, "min_values": None}
    m = re.search(r"values:\s*sets\.(?:New(?:\[string\])?\(([^)]*)\)|Set\[string\]\{\})", expr)
    if m and m.group(1):
        out["values"] = strings(m.group(1))
    for b in ("gte", "lte"):
        m = re.search(rf"\b{b}:\s*(\w+)\.{b}", expr)
        if m:
            d = sym[m.group(1)]
            v = int(d["values"][0])
            out[b] = {"Gt": v + 1, "Gte": v, "Lt": v - 1, "Lte": v}[d["op"]]
    m = re.search(r"MinValues:\s*lo\.ToPtr\((\d+)\)", expr)
    if m:
        out["min_values"] = int(m.group(1))
    return out


def split_args(s):
    args, depth, cur = [], 0, ""
    for ch in s:
        if ch in "({[":
            depth += 1
        if ch in ")}]":
            depth -= 1
        if ch == "," and depth == 0:
            args.append(cur.strip())
            cur = ""
        else:
            cur += ch
    if cur.strip():
        args.append(cur.strip())
    return args


def main():
    src = open(f"{REF}/pkg/scheduling/requirement_test.go").read()
    sym = parse_defs(src)
    out = {"source": "kubernetes-sigs/karpenter @ 7e9d4269 pkg/scheduling/requirement_test.go, requirements_test.go",
           "symbols": sym, "intersection": [], "has": [], "operator": [], "len": [], "compatible": []}
    # tables
    for tm in re.finditer(r'DescribeTable\("([^"]+)",(.*?)\n\t\t\)', src, re.S):
        title, body = tm.group(1), tm.group(2)
        for em in re.finditer(r"Entry\(nil, (.*)\),\s*$", body, re.M):
            args = split_args(em.group(1))
            if "intersect two requirements" in title:
                a, b, exp = args[0], args[1], ", ".join(args[2:])
                e = {"a": a, "b": b}
                if exp.startswith("&Requirement"):
                    e["expected_literal"] = parse_literal(exp, sym)
                else:
                    e["expected_symbol"] = exp
                out["intersection"].append(e)
            elif "right values" in title:
                out["has"].append({"r": args[0], "value": strings(args[1])[0], "expected": "BeTrue" in args[2]})
            elif "operator" in title.lower():
                out["operator"].append({"r": args[0], "expected": OPS[re.search(r"NodeSelectorOp\w+", args[1]).group(0)]})
            elif "len" in title.lower():
                out["len"].append({"r": args[0], "expected": args[1]})
    # Compatible matrices
    src2 = open(f"{REF}/pkg/scheduling/requirements_test.go").read()
    sym2 = parse_defs(src2)
    sym2["unconstrained"] = None
    out["compat_symbols"] = sym2
    for m in re.finditer(r"Expect\((\w+)\.Compatible\((\w+)(, AllowUndefinedWellKnownLabels)?\)\)\.(To|ToNot)\(Succeed\(\)\)",
                         src2):
        a, b, allow, verdict = m.groups()
        if a in sym2 and b in sym2:
            out["compatible"].append({"a": a, "b": b, "allow_undefined": bool(allow), "ok": verdict == "To"})
    json.dump(out, open(f"{sys.argv[2] if len(sys.argv) > 2 else 'tests/golden'}/requirement_kats.json", "w"), indent=0)
    print({k: len(v) for k, v in out.items() if isinstance(v, list)})


if __name__ == "__main__":
    main()
