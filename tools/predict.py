#!/usr/bin/env python
"""The sweep's (exit layer, num_speculations) grid predicted from one scoring pass per prompt
(see layerskip_b200/cli.py: main_predict)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from layerskip_b200.cli import main_predict

if __name__ == "__main__":
    main_predict()
