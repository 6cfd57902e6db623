"""Generates tests/golden/host_loop_traces.json — the engine calls, streamer payloads, stopping-criterion calls and yields of
``generate``, ``generate_batch`` and ``generate_many`` on the recording engine of ``tests/test_cpu_gen_loop.py``, one entry
per case of its matrix. Run:  python tests/golden/make_host_loop_traces.py
"""
import json
import sys
from pathlib import Path

TESTS = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(TESTS.parent), str(TESTS)]
from test_cpu_gen_loop import CASES, GOLDEN, run_case  # noqa: E402


def main():
    out = {name: run_case(name) for name in CASES}
    GOLDEN.write_text(json.dumps(out, separators=(",", ":")) + "\n")
    print(f"wrote {GOLDEN} ({GOLDEN.stat().st_size} bytes, {sum(len(t) for t in out.values())} events)")


if __name__ == "__main__":
    main()
