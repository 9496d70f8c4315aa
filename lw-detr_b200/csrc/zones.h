// Line crossings and zone occupancy per camera stream (lwdetr_zones_*, include/lwdetr_b200.h): one CTA per stream in the
// call, state in a device table allocated once per object.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "records.h"

namespace lwb {

constexpr int ZONE_LINES = 32, ZONE_POLYS = 32, ZONE_POLY_VERTS = 256, ZONE_VERTS = 2048;
constexpr int ZONE_CAPACITY = 4096, ZONE_CLASSES = 1024, ZONE_MAX_OUT = 1024;

struct ZoneHead {                        // per stream
  int32_t frame, n, overflow, pad;       // n records, in index[0, n) by ascending id
};

struct ZoneGeom {                        // per stream; vertices in ZoneTable::verts
  double line[ZONE_LINES][4];
  int32_t n_lines, n_polys;
  int32_t start[ZONE_POLYS + 1];         // polygon p: vertices [start[p], start[p + 1])
};

using ZoneIndex = RecordIndex;           // per record, sorted by id

struct ZoneRec {                         // per slot
  uint32_t inside, side_set, side_pos;   // side of line l: 0 unless bit l of side_set, else +1 / -1 by bit l of side_pos
  int32_t label;
  int32_t entry[ZONE_POLYS];             // entry frame, 0 when outside
};

struct ZoneTable {
  int num_streams, capacity, num_classes, forget_after, zone_anchor, line_anchors;
  ZoneHead* head;                        // [num_streams]
  ZoneGeom* geom;                        // [num_streams]
  double2* verts;                        // [num_streams][ZONE_VERTS]
  ZoneIndex* index;                      // [num_streams][capacity]
  ZoneRec* rec;                          // [num_streams][capacity]
  int32_t* line_counts;                  // [num_streams][ZONE_LINES][num_classes + 1][2]
  int32_t* entries;                      // [num_streams][ZONE_POLYS][num_classes + 1]
};

// streams HOST, B distinct ids in [0, num_streams); everything else DEVICE.  A cudaError_t.
int zones_launch(const ZoneTable& t, const int32_t* ids, const int32_t* labels, const float* boxes, const int32_t* counts, int B, int max_out,
                 const int32_t* streams, uint32_t* inside, int32_t* occupancy, int32_t* events, int max_events, int32_t* event_counts,
                 cudaStream_t st);
// frame back to 1, no records, counters and overflow 0, for n HOST stream ids
int zones_reset_launch(const ZoneTable& t, const int32_t* streams, int n, cudaStream_t st);

}  // namespace lwb
