#!/bin/sh
# TEST-ONLY build of the host emulation of shared arrival lists (see hostemu_pair.cpp).
set -e
cd "$(dirname "$0")"
mkdir -p _build
g++ -O2 -fPIC -shared -std=gnu++17 -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function -Wno-unknown-pragmas \
    -o _build/libdcsim_hostemu_pair.so hostemu_pair.cpp -lm
# the event-loop skeleton of the lane-group GPU builds (warp-uniform: replicas switched off, not broken out of the loop)
g++ -O2 -fPIC -shared -std=gnu++17 -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function -Wno-unknown-pragmas \
    -DDCSIM_HOST_UNIFORM_LOOP -o _build/libdcsim_hostemu_pair_uniform.so hostemu_pair.cpp -lm
