"""Kernel timeline of the LAST step in a chrome trace written by `bench.py --trace` (torch.profiler): per kernel
start offset, duration, stream — to see what overlaps what inside the captured step.
    python scripts/trace_summary.py trace_n2.json"""
import json
import sys


def main(path):
    ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset") and "ts" in e]
    ev.sort(key=lambda e: e["ts"])
    if not ev:
        print("no kernel events")
        return
    # split into steps: a gap > 150 us of GPU idle, or the scan kernel that opens a step
    starts = [i for i, e in enumerate(ev) if "scan_tile_sums" in e["name"] or "Memcpy DtoD" in e["name"]]
    gaps = [0] + [i for i in range(1, len(ev)) if ev[i]["ts"] - max(x["ts"] + x["dur"] for x in ev[max(0, i - 40):i]) > 100]
    b = gaps[-1] if len(gaps) > 1 else 0
    step = ev[b:]
    t0 = step[0]["ts"]
    end = max(e["ts"] + e["dur"] for e in step)
    print(f"{len(step)} GPU events, {end - t0:.1f} us from first start to last end")
    streams = sorted({e["args"].get("stream", 0) for e in step})
    for e in step:
        s = streams.index(e["args"].get("stream", 0))
        print(f"{e['ts'] - t0:9.1f} {e['dur']:8.1f}  s{s}  {e['name'][:90]}")


if __name__ == "__main__":
    main(sys.argv[1])
