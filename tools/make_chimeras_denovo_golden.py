"""Regenerate tests/golden/chimeras_denovo_reference.json: every case of tests/chimeras_denovo_cases.py run through the
reference CLI (oracle/_ref/vsearch --chimeras_denovo ... --threads 1), the sha256 of its input and output files and its
summary counts."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

import chimeras_denovo_cases  # noqa: E402

if __name__ == "__main__":
    chimeras_denovo_cases.make_golden()
