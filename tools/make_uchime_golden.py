"""Regenerate tests/golden/uchime_reference.json: every case of tests/uchime_cases.py run through the reference CLI
(oracle/_ref/vsearch --uchime_ref ... --threads 1), the sha256 of its inputs and output files and its summary counts."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

import uchime_cases  # noqa: E402

if __name__ == "__main__":
    uchime_cases.make_golden()
