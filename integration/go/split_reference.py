#!/usr/bin/env python3
"""Prepares a checkout of spacejam/loghisto for the b200 build tag WITHOUT changing what a plain `go build` compiles.

  python split_reference.py <loghisto checkout> [--dry-run]

The five method bodies the GPU engine replaces -- MetricSystem.Counter, MetricSystem.Histogram, processHistograms,
collectRawMetrics and processMetrics (metrics.go:251-295, 336-387, 420-506 at the surveyed commit) -- are MOVED, text
unchanged, from metrics.go into a new metrics_cpu.go that carries `//go:build !b200`.  Import lists of both files are
trimmed to what each still uses.  Afterwards:

  go build ./...              pure-Go loghisto, byte-for-byte the same functions as before
  go build -tags b200 ./...   the same package with metrics_b200.go (cgo -> libloghisto_b200.so) providing those five methods

Functions are located by name (a `func (ms *MetricSystem) <name>(` line, its doc comment above, the matching closing
brace at column 0), not by line number, so the script survives unrelated edits of metrics.go.
"""
import os
import re
import sys

MOVED = ["Counter", "Histogram", "processHistograms", "collectRawMetrics", "processMetrics"]


def find_function(lines, name):
    """(first, last) line indices of the function, including its doc comment."""
    pat = re.compile(r"^func \(ms \*MetricSystem\) %s\(" % re.escape(name))
    for i, ln in enumerate(lines):
        if pat.match(ln):
            start = i
            while start > 0 and lines[start - 1].startswith("//"):
                start -= 1
            end = i
            while not lines[end].startswith("}"):
                end += 1
            return start, end
    raise SystemExit("metrics.go: func (ms *MetricSystem) %s not found" % name)


def import_block(lines):
    a = next(i for i, ln in enumerate(lines) if ln.startswith("import ("))
    b = next(i for i in range(a, len(lines)) if lines[i].startswith(")"))
    return a, b


def used_imports(import_lines, body):
    keep = []
    for ln in import_lines:
        m = re.search(r'"([^"]+)"', ln)
        if not m:
            if ln.strip() == "" and keep and keep[-1].strip() != "":
                keep.append(ln)
            continue
        pkg = m.group(1).rsplit("/", 1)[-1]
        if re.search(r"\b%s\." % re.escape(pkg), body):
            keep.append(ln)
    while keep and keep[-1].strip() == "":
        keep.pop()
    return keep


def main():
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    root = sys.argv[1]
    dry = "--dry-run" in sys.argv
    src = os.path.join(root, "metrics.go")
    text = open(src).read()
    if "metrics_cpu.go" in text or os.path.exists(os.path.join(root, "metrics_cpu.go")):
        raise SystemExit("already split")
    lines = text.split("\n")
    spans = sorted(find_function(lines, n) for n in MOVED)
    moved, kept, prev = [], [], 0
    for a, b in spans:
        kept += lines[prev:a]
        moved += lines[a:b + 1] + [""]
        prev = b + 1
        while prev < len(lines) and lines[prev].strip() == "":   # the blank line that followed the function
            prev += 1
    kept += lines[prev:]

    ia, ib = import_block(kept)
    header = kept[:ia]                                          # licence comment, package clause
    imports = kept[ia + 1:ib]
    body_kept = "\n".join(kept[ib + 1:])
    body_moved = "\n".join(moved)
    new_metrics = header + ["import ("] + used_imports(imports, body_kept) + [")"] + kept[ib + 1:]
    pkg_line = next(ln for ln in header if ln.startswith("package "))
    licence = []
    for ln in header:
        if ln.startswith("package "):
            break
        licence.append(ln)
    new_cpu = (licence + ["// The pure-Go bodies of the five methods the GPU engine replaces (moved here unchanged from metrics.go by",
                          "// integration/go/split_reference.py of loghisto_b200); compiled unless the b200 build tag is set.", "",
                          "//go:build !b200", "", pkg_line, "", "import ("] + used_imports(imports, body_moved) + [")", ""] + moved)
    out_metrics, out_cpu = "\n".join(new_metrics), "\n".join(new_cpu).rstrip("\n") + "\n"
    n_before = sum(1 for ln in lines if ln.startswith("func "))
    n_after = sum(1 for ln in new_metrics if ln.startswith("func ")) + sum(1 for ln in new_cpu if ln.startswith("func "))
    assert n_before == n_after, (n_before, n_after)
    print("metrics.go: %d -> %d lines; metrics_cpu.go: %d lines (%d functions moved)" %
          (len(lines), len(new_metrics), len(new_cpu), len(MOVED)))
    if dry:
        return
    open(src, "w").write(out_metrics)
    open(os.path.join(root, "metrics_cpu.go"), "w").write(out_cpu)


if __name__ == "__main__":
    main()
