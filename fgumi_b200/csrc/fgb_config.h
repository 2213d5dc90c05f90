// Compile-time geometry shared by the tile planner (host) and the vote kernel (device).
#pragma once
#include <stdint.h>

namespace fgb {

// One CTA = 256 threads, 2 CTAs per SM.  A tile is a run of consecutive units whose byte range in
// each column fits one shared-memory stage.
constexpr int kConsumerWarps = 8;
constexpr int kVoteThreads = kConsumerWarps * 32;        // threads that vote
constexpr int kThreads = kVoteThreads + 32;              // + one TMA producer warp
#ifndef FGB_STAGES
#define FGB_STAGES 2
#endif
#ifndef FGB_TILE_CAP
#define FGB_TILE_CAP 20480
#endif
constexpr int kStages = FGB_STAGES;
constexpr uint32_t kTileCapBytes = FGB_TILE_CAP;  // per column per stage (multiple of 16)
constexpr uint32_t kTileMaxReads = 512;    // read descriptors per stage (8 B each)
constexpr uint32_t kTileMaxUnits = 127;    // unit descriptors per stage (16 B each, +1 sentinel)
#ifndef FGB_WARP_QUEUE_CAP
#define FGB_WARP_QUEUE_CAP 96
#endif
constexpr uint32_t kWarpQueueCap = FGB_WARP_QUEUE_CAP;     // undecided positions buffered per warp per tile
// shallow queues at least this long are resolved one position per lane, shorter ones eight lanes per position
constexpr uint32_t kLaneMinQueue = 24u;
constexpr uint32_t kQtEntries = 256;       // fast-path quality threshold table, indexed by min(n,255)

constexpr uint32_t kTileFlagDirect = 1u;   // unit too large for a stage: kernel reads it from HBM
constexpr uint32_t kTileFlagRegular = 2u;  // all reads one length L, rows back to back at stride
                                           // round_up(L,8), every unit calls L positions (L > 8)
constexpr uint32_t kTileFlagSkew8 = 4u;    // regular tiles: first row starts 8 bytes into the stage
constexpr uint32_t kTileFlagShallow = 8u;  // no unit of the tile has more than 64 reads
// bits 4..5: tile class -- 0 general, 1 shallow (every unit has at most kShallowMax reads), 2 deep (every unit has
// at least kDeepMin reads); tiles are class-homogeneous and each class has its own kernel (vote_kernel.cuh)
constexpr uint32_t kTileClassShift = 4u;
constexpr uint32_t kTileClassMask = 3u << kTileClassShift;
constexpr uint32_t kShallowMax = 4u;
constexpr uint32_t kDeepMin = 24u;
inline uint32_t unit_class(uint32_t n_reads) { return n_reads <= kShallowMax ? 1u : (n_reads >= kDeepMin ? 2u : 0u); }
// bits 8..31: items (8-position words) per unit when uniform over the tile (2..4096), else 0

}  // namespace fgb
