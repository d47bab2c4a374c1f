// retire_moves.h — the move rule of a retirement, shared with transfers: the device ABI (resident_abi.cu), the retire launch
// (device_record.h) and the host mirror (host_mirror.cc) take it from here.  Plain C++, so the host mirror builds without CUDA.
#pragma once
#include <stdint.h>

#include <vector>

namespace bf {

constexpr uint32_t kRetireNoMove = 0xFFFFFFFFu;   // to[i] of a run m + i that leaves rather than moves

// The k-th retired index below m (ascending) receives the k-th live index of [m, m + n); there are as many of each.  to[i] is
// the new index of run m + i, or kRetireNoMove.  -> the number of moves
inline uint32_t retire_moves(const std::vector<uint8_t>& gone, uint32_t m, uint32_t n, std::vector<uint32_t>& to) {
  to.assign(n, kRetireNoMove);
  uint32_t n_moves = 0;
  for (uint32_t i = 0, hole = 0; i < n; ++i) {
    if (gone[m + i]) continue;
    while (!gone[hole]) ++hole;
    to[i] = hole++;
    ++n_moves;
  }
  return n_moves;
}

// the moves of `to` into the caller's arrays (either may be NULL), ascending by target
inline void write_moves(const std::vector<uint32_t>& to, uint32_t m, uint32_t* moves_from, uint32_t* moves_to) {
  for (uint32_t i = 0, k = 0; i < to.size() && (moves_from || moves_to); ++i) {
    if (to[i] == kRetireNoMove) continue;
    if (moves_from) moves_from[k] = m + i;
    if (moves_to) moves_to[k] = to[i];
    ++k;
  }
}

}  // namespace bf
