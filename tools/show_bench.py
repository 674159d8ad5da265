"""print the interesting fields of a bench.py JSON line (file argument)."""
import json
import sys


def main():
    d = json.loads(open(sys.argv[1]).read().strip().splitlines()[-1])
    print(round(d["value"], 1), "clouds/s  e2e", round(d["e2e"]["value"], 1), " ms/step", round(d["ms_per_step"], 3),
          {k: round(v, 3) for k, v in d.get("stage_ms_eager", {}).items()}, d.get("clocks"))


if __name__ == "__main__":
    main()
