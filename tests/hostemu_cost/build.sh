#!/bin/sh
# TEST-ONLY builds of the host emulation with the energy-cost recorder (see hostemu_cost.cpp): plain and the
# warp-uniform event-loop skeleton, with the flags of tests/hostemu/build.sh.
set -e
cd "$(dirname "$0")"
mkdir -p _build
build() {
    g++ -O2 -fPIC -shared -std=gnu++17 -ffp-contract=off -fno-fast-math -Wall -Wno-unused-function -Wno-unknown-pragmas \
        "$@" hostemu_cost.cpp -lm
}
build -o _build/libdcsim_hostemu_cost.so
build -DDCSIM_HOST_UNIFORM_LOOP -o _build/libdcsim_hostemu_cost_uniform.so
