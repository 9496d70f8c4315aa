// Drawing detections, tracks and zones into RGB / NV12 frames in place, with privacy pixelation (lwdetr_annotator_*,
// lwdetr_annotate in include/lwdetr_b200.h; see annotate.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "lwdetr_b200.h"
#include "zones.h"

namespace lwb {

constexpr int ANN_CLASSES = 1024, ANN_K = 1024, ANN_FRAMES = 1024, ANN_PALETTE = 256, ANN_NAME = 32;
constexpr int ANN_GROUP = 32;                                        // frames per launch pair (setup, draw)
constexpr int ANN_TEXT = 64;                                         // bytes of one text slot (the longest label is 49 + NUL)
constexpr int ANN_TEXTS = ANN_K + ZONE_LINES + ZONE_POLYS;           // per frame: one per entry, line and polygon
constexpr int ANN_PRIMS = 4 * ANN_K + ZONE_POLYS + ZONE_VERTS + ZONE_LINES + 2 * (ZONE_LINES + ZONE_POLYS);

// one drawing primitive of a frame, in painter's order in the scratch; [x0, x1) x [y0, y1): its pixels' bounding box in the
// frame (exact for rectangles and texts, conservative for segments and polygons)
struct AnnPrim {
  int32_t x0, y0, x1, y1;
  int32_t kind, alpha;
  uint32_t rgb;                          // R | G << 8 | B << 16
  int32_t p0, p1, p2;                    // segment: line index or -1, vertex a, vertex b; polygon: first vertex, count;
  int32_t pad[2];                        //   text: origin x, y, text slot
};
enum { ANN_PRIV = 0, ANN_FILL = 1, ANN_OUTLINE = 2, ANN_SEG = 3, ANN_POLY = 4, ANN_TEXT_GLYPHS = 5 };

// the object's device tables (one allocation)
struct AnnTable {
  int num_classes;
  uint8_t* palette;                      // [ANN_PALETTE][3]
  int32_t* palette_n;                    // [1]
  char* names;                           // [num_classes][ANN_NAME], NUL-terminated; "" = the id in decimal
  uint8_t* privacy;                      // [num_classes]
  AnnPrim* prims;                        // [ANN_GROUP][ANN_PRIMS]
  int32_t* nprims;                       // [ANN_GROUP][2]: primitives, of which privacy rectangles (first)
  char* texts;                           // [ANN_GROUP][ANN_TEXTS][ANN_TEXT]
};

struct AnnOptions {
  int thickness, text_scale, box_fill_alpha, label, zone_fill_alpha, zone_thickness, privacy_block;
};

// one call's entries and zones; every pointer DEVICE except `streams` (HOST, B stream ids, only read with zones)
struct AnnCall {
  const int32_t* ids;                    // or NULL
  const float* scores;
  const int32_t* labels;
  const float* boxes;
  const int32_t* counts;                 // or NULL
  int k;
  float threshold;
  const ZoneTable* zones;                // or NULL
  const int32_t* streams;
  const int32_t* occupancy;              // [B, 32] or NULL
};

// frames: HOST array of B validated descriptors.  A cudaError_t.
int annotate_launch(const AnnTable& t, const AnnOptions& o, const lwdetr_frame* frames, int B, const AnnCall& c, cudaStream_t st);
int annotate_launch(const AnnTable& t, const AnnOptions& o, const lwdetr_frame_nv12* frames, int B, const AnnCall& c, cudaStream_t st);

}  // namespace lwb
