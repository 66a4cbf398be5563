#!/usr/bin/env python
"""Performance regression gate: compares a fresh `bench.py` JSON line (or an `ep_sweep` / nccl-tests table row set)
with the committed baseline of the same GPU count in profiles/ and fails when a tracked number got worse by more
than the tolerance.  The reference has no automated perf regression check (SURVEY 4: "numbers are pasted into READMEs").

    python bench.py --gpus 1 ... > new1.json
    python scripts/perf_gate.py new1.json                      # baseline: profiles/bench1.json, tolerance 7 %
    python scripts/perf_gate.py new1.json --baseline old.json --tolerance 0.05 --update
"""
import argparse
import json
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (path into the JSON, higher is better)
TRACKED = [
    (("value",), True),
    (("ms_per_step",), False),
    (("dispatch_us",), False),
    (("combine_us",), False),
    (("e2e", "value"), True),
    (("best", "tokens_per_s"), True),
]


def load_line(path):
    txt = open(path).read().strip()
    try:
        return json.loads(txt)
    except json.JSONDecodeError:
        for line in reversed(txt.splitlines()):
            if line.startswith("{"):
                return json.loads(line)
    raise SystemExit(f"{path}: no JSON object found")


def get(d, path):
    for k in path:
        if not isinstance(d, dict) or k not in d:
            return None
        d = d[k]
    return d if isinstance(d, (int, float)) else None


def compare(new, old, tol):
    rows, failed = [], False
    for path, hib in TRACKED:
        a, b = get(new, path), get(old, path)
        if a is None or b is None or b == 0:
            continue
        change = (a - b) / abs(b)
        worse = (-change if hib else change) > tol
        failed |= worse
        rows.append((".".join(path), b, a, change, "REGRESSION" if worse else "ok"))
    # per-CTA-count sweep, matched by num_sms
    olds = {r.get("num_sms"): r for r in old.get("sm_sweep", []) if isinstance(r, dict)}
    for r in new.get("sm_sweep", []):
        o = olds.get(r.get("num_sms"))
        if not o:
            continue
        for k in ("dispatch_us", "combine_us"):
            if k in r and k in o and o[k]:
                change = (r[k] - o[k]) / o[k]
                worse = change > tol
                failed |= worse
                rows.append((f"sm_sweep[{r['num_sms']}].{k}", o[k], r[k], change, "REGRESSION" if worse else "ok"))
    return rows, failed


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("new")
    ap.add_argument("--baseline", default=None)
    ap.add_argument("--tolerance", type=float, default=0.07, help="relative worsening that fails the gate (default 7 %%)")
    ap.add_argument("--update", action="store_true", help="on success, the new file becomes the baseline")
    a = ap.parse_args(argv)
    new = load_line(a.new)
    if new.get("unavailable"):
        raise SystemExit(f"{a.new}: arm unavailable: {new['unavailable']}")
    base = a.baseline or os.path.join(ROOT, "profiles", f"bench{int(new.get('n_gpus', 1))}.json")
    if not os.path.exists(base):
        raise SystemExit(f"no baseline {base}")
    old = load_line(base)
    for k in ("metric", "unit"):
        if new.get(k) != old.get(k):
            raise SystemExit(f"{k} differs: {new.get(k)!r} vs baseline {old.get(k)!r}")
    if new.get("config", {}).get("num_sms") != old.get("config", {}).get("num_sms"):
        print(f"note: headline CTA count differs ({new.get('config', {}).get('num_sms')} vs {old.get('config', {}).get('num_sms')})")
    rows, failed = compare(new, old, a.tolerance)
    w = max(len(r[0]) for r in rows) if rows else 10
    for name, b, v, ch, verdict in rows:
        print(f"{name:<{w}}  baseline {b:>14.4g}  new {v:>14.4g}  {ch * 100:+7.2f} %  {verdict}")
    reasons = (new.get("clocks") or {}).get("reasons") or []
    if any("thermal" in str(r) or "hw_slowdown" in str(r) for r in reasons):
        print("note: the new run was throttled:", reasons)
    if failed:
        print(f"FAILED: at least one tracked number is more than {a.tolerance * 100:.0f} % worse than {os.path.relpath(base, ROOT)}")
        return 1
    print("passed")
    if a.update:
        shutil.copyfile(a.new, base)
        print("baseline updated:", base)
    return 0


if __name__ == "__main__":
    sys.exit(main())
