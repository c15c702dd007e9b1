#!/bin/sh
# TEST-ONLY build of the oracle's created-job record (see oracle_tail.c); the oracle's own flags (oracle/Makefile).
set -e
cd "$(dirname "$0")"
mkdir -p _build
gcc -O2 -fPIC -shared -std=gnu11 -ffp-contract=off -fno-fast-math -fopenmp \
    -fno-builtin-log -fno-builtin-exp -fno-builtin-pow -fno-builtin-sin -fno-builtin-sqrt -Wall -Wextra \
    -o _build/liboracle_tail.so oracle_tail.c -lm
