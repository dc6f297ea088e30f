/* TEST DOUBLE (tests only, never shipped): the record writers of the mock_*.c test doubles of the C ABI.  A recorded call
 * appends "call <name>" and then one "<array> <n> v0 v1 ..." line per array to the file named by $MOCK_DUMP (n = 0 for a
 * null array; without $MOCK_DUMP the records go to /dev/null).  Doubles are written with 17 significant digits, so that
 * the tests read back exactly what the shim passed. */
#ifndef MOCK_DUMP_H
#define MOCK_DUMP_H
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

static inline FILE* mock_dump_open(void) {
  const char* p = getenv("MOCK_DUMP");
  return fopen(p ? p : "/dev/null", "a");
}
/* a call recorded without arrays */
static inline void dump_call(const char* name) {
  FILE* f = mock_dump_open();
  fprintf(f, "call %s\n", name);
  fclose(f);
}

#define MOCK_DUMP_WRITER(NAME, T, FMT, CAST)                                  \
  static inline void NAME(FILE* f, const char* name, const T* v, long long n) { \
    fprintf(f, "%s %lld", name, v ? n : 0);                                   \
    for (long long i = 0; v && i < n; ++i) fprintf(f, FMT, (CAST)v[i]);       \
    fprintf(f, "\n");                                                         \
  }
MOCK_DUMP_WRITER(dump_i32, int32_t, " %d", int)
MOCK_DUMP_WRITER(dump_i64, int64_t, " %lld", long long)
MOCK_DUMP_WRITER(dump_u8, uint8_t, " %d", int)
MOCK_DUMP_WRITER(dump_u16, uint16_t, " %u", unsigned)
MOCK_DUMP_WRITER(dump_u32, uint32_t, " %u", unsigned)
MOCK_DUMP_WRITER(dump_u64, uint64_t, " %llu", unsigned long long)
MOCK_DUMP_WRITER(dump_f64, double, " %.17g", double)
#undef MOCK_DUMP_WRITER

#endif
