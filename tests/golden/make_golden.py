#!/usr/bin/env python3
"""Transcribe the reference's known-answer tests into JSON fixtures.

The reference (mwhittaker/frankenpaxos) is Scala and cannot be compiled or run
in this environment (no JVM / sbt / network), so its scalatest files are read AS
DATA: every deterministic assertion of the helper classes on the quorum-vote
path is parsed out of the test sources and written to tests/golden/*.json as a
list of operations + expectations.  tests/test_golden_oracle.py replays them
against oracle/fpx_oracle.cc; the `-m gpu` tests replay the quorum vectors
against the CUDA predicates.

Needs a checkout of the reference; the JSON fixtures are committed, the tests never run this:
    FPX_REFERENCE=<reference checkout> python tests/golden/make_golden.py
Sources (relative to the reference root), shared/src/test/scala/:
    quorums/GridTest.scala            :11-102
    quorums/SimpleMajorityTest.scala  :11-63
    quorums/UnanimousWrites.scala     :11-75
    compact/IntPrefixSetTest.scala    :25-94, 105-127, 150-172, 273-294
    roundsystem/RoundSystemTest.scala :8-62   (ClassicRoundRobin only)
    util/TopOneTest.scala             :15-86
    util/QuorumWatermarkTest.scala    :7-40
    util/BufferMapTest.scala
scalacheck `forAll` property blocks are NOT transcribed (they have no fixed
vectors); tests/test_oracle_properties.py re-expresses them with hypothesis
using the same generator ranges (IntPrefixSetTest.scala:15-23).
"""
import itertools
import json
import os
import re
import sys

REF = os.environ.get("FPX_REFERENCE", "")
T = os.path.join(REF, "shared/src/test/scala")
OUT = os.path.dirname(os.path.abspath(__file__))


def read(rel):
    with open(os.path.join(T, rel)) as f:
        return f.read().split("\n")


def ints(s):
    s = s.strip()
    return [int(x) for x in s.split(",")] if s else []


def test_blocks(lines):
    """Yield (name, first_line_no, body_lines) for every `... in {` block."""
    i = 0
    while i < len(lines):
        m = re.search(r'(?:should|it should|should)\s+"([^"]+)"\s+in\s*\{', lines[i])
        if not m and re.search(r'"\s*in\s*\{\s*$', lines[i]):
            m = re.search(r'"([^"]+)"\s+in\s*\{', lines[i])
        if m:
            name = m.group(1)
            depth = lines[i].count("{") - lines[i].count("}")
            body = []
            j = i + 1
            while j < len(lines) and depth > 0:
                depth += lines[j].count("{") - lines[j].count("}")
                if depth > 0:
                    body.append((j + 1, lines[j]))
                j += 1
            yield name, i + 1, body
            i = j
        else:
            i += 1


# --------------------------------------------------------------------------- quorums
def parse_quorums():
    res = {}
    specs = [
        ("grid", "quorums/GridTest.scala", r"new Grid\((Seq\(.*\))\)"),
        ("simple_majority", "quorums/SimpleMajorityTest.scala", r"new SimpleMajority\(Set\((.*?)\)\)"),
        ("unanimous_writes", "quorums/UnanimousWrites.scala", r"new UnanimousWrites\(Set\((.*?)\)\)"),
    ]
    for key, rel, ctor in specs:
        lines = read(rel)
        cases = []
        members = None
        for name, lineno, body in test_blocks(lines):
            loops = []
            for ln, line in body:
                m = re.search(ctor, line)
                if m:
                    raw = m.group(1)
                    if key == "grid":
                        rows = re.findall(r"Seq\(([\d,\s]+)\)", raw)
                        members = [ints(r) for r in rows]
                    else:
                        members = ints(raw)
                    continue
                m = re.match(r"\s*for\s*\((.*)\)\s*\{", line)
                if m:
                    vars_, ranges = [], []
                    for g in m.group(1).split(";"):
                        mm = re.match(r"\s*(\w+)\s*<-\s*(-?\d+)\s+to\s+(-?\d+)", g)
                        vars_.append(mm.group(1))
                        ranges.append(range(int(mm.group(2)), int(mm.group(3)) + 1))
                    loops.append((vars_, ranges))
                    continue
                if line.strip() == "}" and loops:
                    loops.pop()
                    continue
                m = re.search(r"qs\.(\w+)\(Set\((.*?)\)\)\s+shouldBe\s+(true|false)", line)
                if m:
                    pred, elems, exp = m.group(1), m.group(2), m.group(3) == "true"
                    all_vars = [v for vs, _ in loops for v in vs]
                    all_ranges = [r for _, rs in loops for r in rs]
                    combos = itertools.product(*all_ranges) if all_vars else [()]
                    for combo in combos:
                        env = dict(zip(all_vars, combo))
                        xs = sorted(set(int(eval(e, {}, env)) for e in elems.split(",") if e.strip()))
                        cases.append({"pred": pred, "set": xs, "expect": exp, "line": ln})
        res[key] = {"source": "shared/src/test/scala/" + rel, "members": members, "cases": cases}
    return res


# --------------------------------------------------------------------------- op scripts
def set_lit(s):
    m = re.match(r"Set\((.*)\)", s.strip())
    return ints(m.group(1))


def parse_ips():
    lines = read("compact/IntPrefixSetTest.scala")
    tests = []
    for name, lineno, body in test_blocks(lines):
        text = "\n".join(l for _, l in body)
        if "forAll" in text:
            continue  # property test, see test_oracle_properties.py
        ops = []
        for ln, line in body:
            s = line.strip()
            if not s or s.startswith("//"):
                continue
            m = re.match(r"val (\w+) = IntPrefixSet\(\)$", s)
            if m:
                ops.append(["new", m.group(1)]); continue
            m = re.match(r"val (\w+) = IntPrefixSet\((Set\(.*\))\)$", s)
            if m:
                ops.append(["from_set", m.group(1), set_lit(m.group(2))]); continue
            m = re.match(r"val (\w+) = (\w+)\.(union|diff)\((\w+)\)$", s)
            if m:
                ops.append([m.group(3), m.group(1), m.group(2), m.group(4)]); continue
            m = re.match(r"val (\w+) = (\w+)\.clone\(\)$", s)
            if m:
                ops.append(["clone", m.group(1), m.group(2)]); continue
            m = re.match(r"val (\w+) = (\w+)\.diffIterator\((\w+)\)$", s)
            if m:
                ops.append(["diff_iterator", m.group(1), m.group(2), m.group(3)]); continue
            m = re.match(r"(\w+)\.(add|subtractOne)\((-?\d+)\)$", s)
            if m:
                ops.append([m.group(2), m.group(1), int(m.group(3))]); continue
            m = re.match(r"(\w+)\.addAll\(IntPrefixSet\((Set\(.*\))\)\)$", s)
            if m:
                ops.append(["add_all_set", m.group(1), set_lit(m.group(2))]); continue
            m = re.match(r"(\w+)\.contains\((-?\d+)\) shouldBe (true|false)$", s)
            if m:
                ops.append(["expect_contains", m.group(1), int(m.group(2)), m.group(3) == "true", ln]); continue
            m = re.match(r"(\w+)\.materialize\(\) shouldBe (Set\(.*\))$", s)
            if m:
                ops.append(["expect_materialize", m.group(1), set_lit(m.group(2)), ln]); continue
            m = re.match(r"(\w+)\.getWatermark\(\) shouldBe (-?\d+)$", s)
            if m:
                ops.append(["expect_watermark", m.group(1), int(m.group(2)), ln]); continue
            m = re.match(r"(\w+) shouldBe IntPrefixSet\((Set\(.*\))\)$", s)
            if m:
                ops.append(["expect_equals_set", m.group(1), set_lit(m.group(2)), ln]); continue
            m = re.match(r"(\w+)\.hasNext shouldBe (true|false)$", s)
            if m:
                ops.append(["expect_has_next", m.group(1), m.group(2) == "true", ln]); continue
            m = re.match(r"(\w+)\.next\(\) shouldBe (-?\d+)$", s)
            if m:
                ops.append(["expect_next", m.group(1), int(m.group(2)), ln]); continue
            raise SystemExit(f"IntPrefixSetTest.scala:{ln}: unparsed line: {s}")
        tests.append({"name": name, "line": lineno, "ops": ops})
    return {"source": "shared/src/test/scala/compact/IntPrefixSetTest.scala", "tests": tests}


def parse_roundsystem():
    lines = read("roundsystem/RoundSystemTest.scala")
    cases = []
    n = None
    for ln, line in enumerate(lines, 1):
        if "ClassicStutteredRoundRobin" in line or "RoundZeroFast" in line or "MixedRoundRobin" in line:
            break  # only the ClassicRoundRobin section
        m = re.search(r"new RoundSystem\.ClassicRoundRobin\((\d+)\)", line)
        if m:
            n = int(m.group(1)); continue
        m = re.search(r"rs\.leader\((-?\d+)\) shouldBe (-?\d+)", line)
        if m:
            cases.append({"op": "leader", "n": n, "round": int(m.group(1)), "expect": int(m.group(2)), "line": ln}); continue
        m = re.search(r"rs\.nextClassicRound\(leaderIndex = (-?\d+), round = (-?\d+)\) shouldBe (-?\d+)", line)
        if m:
            cases.append({"op": "nextClassicRound", "n": n, "leader": int(m.group(1)), "round": int(m.group(2)),
                          "expect": int(m.group(3)), "line": ln})
    return {"source": "shared/src/test/scala/roundsystem/RoundSystemTest.scala", "cases": cases}


def parse_topone():
    lines = read("util/TopOneTest.scala")
    tests = []
    for name, lineno, body in test_blocks(lines):
        ops = []
        for ln, line in body:
            s = line.strip()
            if not s:
                continue
            m = re.match(r"val (\w+) = new TopOne\((\d+), like\)$", s)
            if m:
                ops.append(["new", m.group(1), int(m.group(2))]); continue
            m = re.match(r"(\w+)\.put\(\((\d+), (\d+)\)\)$", s)
            if m:
                ops.append(["put", m.group(1), int(m.group(2)), int(m.group(3))]); continue
            m = re.match(r"(\w+)\.mergeEquals\((\w+)\)$", s)
            if m:
                ops.append(["merge", m.group(1), m.group(2)]); continue
            m = re.match(r"(\w+)\.get\(\) shouldBe mutable\.Buffer\((.*)\)$", s)
            if m:
                ops.append(["expect_get", m.group(1), ints(m.group(2)), ln]); continue
            raise SystemExit(f"TopOneTest.scala:{ln}: unparsed line: {s}")
        tests.append({"name": name, "line": lineno, "ops": ops})
    return {"source": "shared/src/test/scala/util/TopOneTest.scala", "tests": tests}


def parse_quorum_watermark():
    lines = read("util/QuorumWatermarkTest.scala")
    tests = []
    for name, lineno, body in test_blocks(lines):
        ops = []
        for ln, line in body:
            s = line.split("//")[0].strip()
            if not s:
                continue
            m = re.match(r"val (\w+) = new QuorumWatermark\(numWatermarks = (\d+)\)$", s)
            if m:
                ops.append(["new", int(m.group(2))]); continue
            m = re.match(r"watermark\.update\((\d+), (\d+)\)$", s)
            if m:
                ops.append(["update", int(m.group(1)), int(m.group(2))]); continue
            m = re.match(r"watermark\.watermark\((\d+)\) shouldBe (\d+)$", s)
            if m:
                ops.append(["expect_watermark", int(m.group(1)), int(m.group(2)), ln]); continue
            raise SystemExit(f"QuorumWatermarkTest.scala:{ln}: unparsed line: {s}")
        tests.append({"name": name, "line": lineno, "ops": ops})
    return {"source": "shared/src/test/scala/util/QuorumWatermarkTest.scala", "tests": tests}


def parse_buffermap():
    lines = read("util/BufferMapTest.scala")
    tests = []
    for name, lineno, body in test_blocks(lines):
        ops = []
        ok = True
        for ln, line in body:
            s = line.strip()
            if not s:
                continue
            m = re.match(r"val map = new BufferMap\[String\]\((\d+)\)$", s)
            if m:
                ops.append(["new", int(m.group(1))]); continue
            m = re.match(r'map\.put\((\d+), "(\d+)"\)$', s)
            if m:
                ops.append(["put", int(m.group(1)), int(m.group(2))]); continue
            m = re.match(r"map\.garbageCollect\((\d+)\)$", s)
            if m:
                ops.append(["gc", int(m.group(1))]); continue
            m = re.match(r"map\.get\((\d+)\) shouldBe None$", s)
            if m:
                ops.append(["expect_get", int(m.group(1)), -1, ln]); continue
            m = re.match(r'map\.get\((\d+)\) shouldBe Some\("(\d+)"\)$', s)
            if m:
                ops.append(["expect_get", int(m.group(1)), int(m.group(2)), ln]); continue
            ok = False  # iterator / toMap tests: not on the path
            break
        if ok and ops:
            tests.append({"name": name, "line": lineno, "ops": ops})
    return {"source": "shared/src/test/scala/util/BufferMapTest.scala", "tests": tests}


def main():
    if not os.path.isdir(T):
        sys.exit(f"reference tests not found at {T}")
    data = {
        "quorums.json": parse_quorums(),
        "int_prefix_set.json": parse_ips(),
        "round_system.json": parse_roundsystem(),
        "top_one.json": parse_topone(),
        "quorum_watermark.json": parse_quorum_watermark(),
        "buffer_map.json": parse_buffermap(),
    }
    for name, d in data.items():
        with open(os.path.join(OUT, name), "w") as f:
            json.dump(d, f, indent=1, sort_keys=True)
            f.write("\n")
    q = data["quorums.json"]
    print({k: len(v["cases"]) for k, v in q.items()},
          "ips tests", len(data["int_prefix_set.json"]["tests"]),
          "rr", len(data["round_system.json"]["cases"]),
          "topone", len(data["top_one.json"]["tests"]),
          "qw", len(data["quorum_watermark.json"]["tests"]),
          "bm", len(data["buffer_map.json"]["tests"]))


if __name__ == "__main__":
    main()
