#!/bin/sh
# TEST-ONLY builds of the oracle's per-job instants (oracle_jobs.c) and per-arrival record (oracle_lists.c); the oracle's own flags
# (oracle/Makefile).
set -e
cd "$(dirname "$0")"
mkdir -p _build
gcc -O2 -fPIC -shared -std=gnu11 -ffp-contract=off -fno-fast-math -fopenmp \
    -fno-builtin-log -fno-builtin-exp -fno-builtin-pow -fno-builtin-sin -fno-builtin-sqrt -Wall -Wextra \
    -o _build/liboracle_jobs.so oracle_jobs.c -lm
# the oracle's per-arrival record (see oracle_lists.c), same flags
gcc -O2 -fPIC -shared -std=gnu11 -ffp-contract=off -fno-fast-math -fopenmp \
    -fno-builtin-log -fno-builtin-exp -fno-builtin-pow -fno-builtin-sin -fno-builtin-sqrt -Wall -Wextra \
    -o _build/liboracle_lists.so oracle_lists.c -lm
