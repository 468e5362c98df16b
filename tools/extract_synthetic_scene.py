#!/usr/bin/env python
"""Extracts the reference's synthetic courtyard sequence (config/synthetic/courtyard.yaml, the workload of
BASELINE.json configs[0]) into tests/golden/synthetic_courtyard.json: the dict the YAML parses to, with its values as
numbers, so that the tests and Binding.synthetic_sequence need no YAML parser.

An empty YAML key (`lines:` with no items) parses to null and is written as an empty list.

usage: python tools/extract_synthetic_scene.py [/root/reference] [out.json]
tests/test_synthetic_oracle.py checks the file's shape."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_OUT = os.path.join(ROOT, "tests", "golden", "synthetic_courtyard.json")


def extract(reference="/root/reference"):
    import yaml   # only here: the package and the tests read the JSON
    with open(os.path.join(reference, "config", "synthetic", "courtyard.yaml")) as f:
        spec = yaml.safe_load(f)
    acq = spec["acquisition"]
    for key in ("triangles", "lines", "spheres", "balls"):
        acq[key] = acq.get(key) or []
    return spec


def main(argv):
    reference = argv[1] if len(argv) > 1 else "/root/reference"
    out = argv[2] if len(argv) > 2 else DEFAULT_OUT
    with open(out, "w") as f:
        json.dump(extract(reference), f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", out)


if __name__ == "__main__":
    main(sys.argv)
