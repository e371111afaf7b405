#!/usr/bin/env python
"""Per-exit-layer perplexity and greedy agreement with full depth (see layerskip_b200/cli.py: main_score)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from layerskip_b200.cli import main_score

if __name__ == "__main__":
    main_score()
