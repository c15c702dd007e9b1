#!/bin/sh
# TEST-ONLY build of the host emulation with the job-resources recorder (see hostemu_jres.cpp).
set -e
cd "$(dirname "$0")"
mkdir -p _build
g++ -O2 -fPIC -shared -std=gnu++17 -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function -Wno-unknown-pragmas \
    -o _build/libdcsim_hostemu_jres.so hostemu_jres.cpp -lm
# the event-loop skeleton of the lane-group GPU builds (warp-uniform: replicas switched off, not broken out of the loop)
g++ -O2 -fPIC -shared -std=gnu++17 -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function -Wno-unknown-pragmas \
    -DDCSIM_HOST_UNIFORM_LOOP -o _build/libdcsim_hostemu_jres_uniform.so hostemu_jres.cpp -lm
