#!/bin/sh
# TEST-ONLY build of the host emulation with the job-log ensemble recorder (see hostemu_jens.cpp).
set -e
cd "$(dirname "$0")"
mkdir -p _build
g++ -O2 -fPIC -shared -std=gnu++17 -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function -Wno-unknown-pragmas \
    -o _build/libdcsim_hostemu_jens.so hostemu_jens.cpp -lm
# the event-loop skeleton of the lane-group GPU builds (warp-uniform: replicas switched off, not broken out of the loop)
g++ -O2 -fPIC -shared -std=gnu++17 -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function -Wno-unknown-pragmas \
    -DDCSIM_HOST_UNIFORM_LOOP -o _build/libdcsim_hostemu_jens_uniform.so hostemu_jens.cpp -lm
