/*
 * TEST-ONLY.  The oracle probes of the CPU tests in one library: the C oracle (oracle/dcsim_oracle.c, unchanged) and,
 * on top of it, the per-job instants (oracle_jobs.c), the per-arrival record (oracle_lists.c), the occupancy checkers
 * (oracle_occ.c), every created job (oracle_tail.c), the power profile (oracle_power.c) and the energy cost
 * (oracle_cost.c).  Nothing here is part of, linked into, or reachable from the product library.  The oracle's tie hook
 * is its own dcoracle_set_test_time_quantum.
 */
#include "../../oracle/dcsim_oracle.c"

#include "oracle_jobs.c"
#include "oracle_lists.c"
#include "oracle_occ.c"
#include "oracle_tail.c"
#include "oracle_power.c"
#include "oracle_cost.c"
