#!/bin/sh
# TEST-ONLY build of the energy-cost oracle probe (see oracle_cost.c); the oracle's own flags (oracle/Makefile).
set -e
cd "$(dirname "$0")"
mkdir -p _build
gcc -O2 -fPIC -shared -std=gnu11 -ffp-contract=off -fno-fast-math -fopenmp \
    -fno-builtin-log -fno-builtin-exp -fno-builtin-pow -fno-builtin-sin -fno-builtin-sqrt -Wall -Wextra \
    -o _build/liboracle_cost.so oracle_cost.c -lm
