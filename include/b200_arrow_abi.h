/* Arrow C Data Interface structs (https://arrow.apache.org/docs/format/CDataInterface.html).
 * This is the ABI-stable layout both arrow-rs (`arrow::ffi::FFI_ArrowArray/FFI_ArrowSchema`)
 * and pyarrow (`_export_to_c`) produce; the engine's C-ABI exchanges all column data
 * with the host through these structs (SURVEY.md §8(b), last row).                      */
#ifndef B200_ARROW_ABI_H
#define B200_ARROW_ABI_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#ifndef ARROW_C_DATA_INTERFACE
#define ARROW_C_DATA_INTERFACE
#define ARROW_FLAG_DICTIONARY_ORDERED 1
#define ARROW_FLAG_NULLABLE 2
#define ARROW_FLAG_MAP_KEYS_SORTED 4

struct ArrowSchema {
  const char* format;
  const char* name;
  const char* metadata;
  int64_t flags;
  int64_t n_children;
  struct ArrowSchema** children;
  struct ArrowSchema* dictionary;
  void (*release)(struct ArrowSchema*);
  void* private_data;
};

struct ArrowArray {
  int64_t length;
  int64_t null_count;
  int64_t offset;
  int64_t n_buffers;
  int64_t n_children;
  const void** buffers;
  struct ArrowArray** children;
  struct ArrowArray* dictionary;
  void (*release)(struct ArrowArray*);
  void* private_data;
};
#endif /* ARROW_C_DATA_INTERFACE */

#ifdef __cplusplus
}
#endif
#endif
