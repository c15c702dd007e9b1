#!/bin/sh
# TEST-ONLY builds of the single-lane host emulation of the device core (see hostemu.cpp).
set -e
cd "$(dirname "$0")"
mkdir -p _build
build() {
    g++ -O2 -fPIC -shared -std=gnu++17 -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function -Wno-unknown-pragmas \
        "$@" hostemu.cpp -lm
}
build -o _build/libdcsim_hostemu.so
# the event-loop skeleton of the lane-group GPU builds (warp-uniform: replicas are switched off, not broken out of the
# loop; budget and status handled through the `on` flag) compiled for the host's single lane
build -DDCSIM_HOST_UNIFORM_LOOP -o _build/libdcsim_hostemu_uniform.so
# conditioning probe: every 5th pow() result moved by one ulp
build -DDCSIM_HOSTEMU_PERTURB -o _build/libdcsim_hostemu_perturbed.so
# the list merge with a ring of one chunk only: every scan that reaches back or ahead takes the HBM fall-back path
build -DDCSIM_MERGE_RING=32u -o _build/libdcsim_hostemu_smallring.so
