// The summation order of the bit-reproducible weight gradients (temporal_entry.cu, causal_conv.cu): the pixel tiles, numbered in a
// fixed order, are cut into c = min(tiles, WG_MAX_CHUNKS) chunks, chunk i holding tiles [i * tiles / c, (i + 1) * tiles / c); each
// chunk stores its partial and a reduce kernel adds the partials in ascending chunk order.  The chunk count is a constant, not the SM
// count, so the order depends on the shape only.
#pragma once

namespace fiery {

constexpr int WG_MAX_CHUNKS = 128;

inline int wgrad_chunks(long long tiles) { return static_cast<int>(tiles < WG_MAX_CHUNKS ? tiles : WG_MAX_CHUNKS); }

}  // namespace fiery
