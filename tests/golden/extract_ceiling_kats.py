"""Extracts the request-ceiling known-answer tests of the reference (pkg/utils/resources/suite_test.go:40-651, "Resource
Calculations") into tests/golden/ceiling_kats.json: for every It(...) the pod (container requests / limits, init
containers in order with their restart policy, RuntimeClass overhead, pod-level resources) and the expected
resources.Ceiling(pod).Requests / .Limits.  Run against a checkout of the reference; the JSON is committed.

    python tests/golden/extract_ceiling_kats.py <reference checkout>
"""
import json
import os
import re
import sys

SRC = os.path.join(sys.argv[1], "pkg/utils/resources/suite_test.go")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ceiling_kats.json")


def block(s, i):
    """text of the brace-balanced block whose '{' is at or after s[i]; returns (inner, index after the closing brace)"""
    j = s.index("{", i)
    depth, k = 0, j
    while True:
        if s[k] == "{":
            depth += 1
        elif s[k] == "}":
            depth -= 1
            if depth == 0:
                return s[j + 1:k], k + 1
        k += 1


def resource_list(text):
    return {m.group(1).lower(): m.group(2) for m in re.finditer(r'v1\.Resource(\w+):\s*resource\.MustParse\("([^"]+)"\)', text)}


def requirements(text):
    out = {"requests": {}, "limits": {}}
    for side in ("Requests", "Limits"):
        m = re.search(side + r":\s*v1\.ResourceList", text)
        if m:
            inner, _ = block(text, m.end())
            out[side.lower()] = resource_list(inner)
    return out


def top_level_field(text, name):
    """the brace block of `name:` at nesting depth 0 of `text` (PodOptions fields only, not the containers' own)"""
    depth = 0
    for m in re.finditer(r"[{}]|" + re.escape(name) + r":", text):
        tok = m.group(0)
        if tok == "{":
            depth += 1
        elif tok == "}":
            depth -= 1
        elif depth == 0 and (m.start() == 0 or not (text[m.start() - 1].isalnum())):
            inner, _ = block(text, m.end())
            return inner
    return None


def main():
    src = open(SRC).read()
    kats = []
    for m in re.finditer(r'\bIt\("([^"]+)", func\(\) \{', src):
        body, _ = block(src, m.end() - 1)
        if "resources.Ceiling(pod)" not in body:
            continue
        po = re.search(r"test\.PodOptions", body)
        opts, _ = block(body, po.end())
        pod = {"requests": {}, "limits": {}, "init_containers": [], "overhead": {}, "pod_level_requests": {}, "pod_level_limits": {}}
        rr = top_level_field(opts, "ResourceRequirements")
        if rr is not None:
            r = requirements(rr)
            pod["requests"], pod["limits"] = r["requests"], r["limits"]
        pr = top_level_field(opts, "PodResourceRequirements")
        if pr is not None:
            r = requirements(pr)
            pod["pod_level_requests"], pod["pod_level_limits"] = r["requests"], r["limits"]
        ov = top_level_field(opts, "Overhead")
        if ov is not None:
            pod["overhead"] = resource_list(ov)
        ic = top_level_field(opts, "InitContainers")
        if ic is not None:
            i = 0
            while True:
                try:
                    inner, i = block(ic, i)
                except ValueError:
                    break
                r = requirements(inner)
                pod["init_containers"].append({"restart_always": "ContainerRestartPolicyAlways" in inner,
                                               "requests": r["requests"], "limits": r["limits"]})
        exp = {}
        for side in ("Requests", "Limits"):
            e = re.search(r"ExpectResources\(podResources\." + side + r",\s*v1\.ResourceList", body)
            inner, _ = block(body, e.end())
            exp[side.lower()] = resource_list(inner)
        line = src[:m.start()].count("\n") + 1
        kats.append({"name": m.group(1), "line": line, "pod": pod, "expected": exp})
    json.dump({"source": "pkg/utils/resources/suite_test.go:40-651", "cases": kats}, open(OUT, "w"), indent=1)
    print(len(kats), "cases ->", OUT)


if __name__ == "__main__":
    main()
