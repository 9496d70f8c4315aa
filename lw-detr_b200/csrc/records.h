// The index entry of a per-stream record table (lwdetr_zones, lwdetr_speed): one per record, sorted by id, pointing at the
// record's fixed slot.  Kept apart from the kernels' device code so that the C ABI layer can read it back.
#pragma once
#include <stdint.h>

namespace lwb {

struct RecordIndex {
  int32_t id, slot, last_seen;
};

}  // namespace lwb
