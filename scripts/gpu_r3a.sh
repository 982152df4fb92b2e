#!/bin/bash
timeout 1200 python -m pytest tests -m gpu -x -q 2>&1 | tail -4
