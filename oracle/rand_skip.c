/*
 * n draws of the C library's rand(): the rand_skip of oracle/fa_ref.py, which may pass 2^32 (one ctypes call per draw cannot).
 * rand() keeps one state per process, so these draws advance the generator that the compiled reference shuffles with.  A library
 * of its own (oracle/_build/librand_skip.so), built from this file alone, so that it is there whether or not the reference's
 * sources were available when oracle/_ref/ was built.  TEST INFRASTRUCTURE ONLY.
 */
#include <stdint.h>
#include <stdlib.h>

void fa_ref_skip_rand(uint64_t n) {
    while (n--) (void)rand();
}
