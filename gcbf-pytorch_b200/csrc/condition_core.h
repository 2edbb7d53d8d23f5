// Per-element pieces of the CBF-condition field's two-hop probe graphs (condition_kernels.cuh), written once for device and host:
// tests/host_driver/condition_grid.cpp compiles them with g++ -ffp-contract=off for the CPU test-suite.
//
// A probe t (numbered as in field_core.h) is graph b's agent a moved to s'_t.  h_dot of a needs x_dot at a and at every agent source
// j of a's in-edges, and x_dot_j needs the actor's u_j, which reads j's own in-edges.  So a probe becomes these rows of a chunk:
//   a'  row i of the chunk's first Tc rows: the moved agent, with a's in-edges in G' (the graph with a moved);
//   j'  one row per agent source j of a', in a'-edge order: a copy of j's unmoved state, with j's in-edges in G';
// followed by the original nodes at rows src_off + (b * N + k).  Sources are mapped to rows by cond_source_row: an agent source of
// a' is its j' row, a source a of a j' row is the a' row, every other source is the original node's row.
#pragma once
#include "field_core.h"

namespace gcbf {
namespace cond {

// kind of a probe row (the rows export of gcbf_cbf_condition_probe_fill)
constexpr int kRowMoved = 0;      // a'
constexpr int kRowNeighbour = 1;  // j'

// row of source `src` (node id in the given graphs) of an edge into a probe row.  a_node: the probed agent's node id; a_row: its a'
// row; j_row: the j' row if src is an agent source of a' (target_is_moved), else unused.
GCBF_GHD int64_t cond_source_row(int64_t src, int64_t a_node, bool target_is_moved, bool src_is_agent, int64_t a_row, int64_t j_row,
                                  int64_t src_off) {
  if (target_is_moved) return src_is_agent ? j_row : src_off + src;
  return src == a_node ? a_row : src_off + src;
}

// the state a source contributes to G': the moved state for a, the given state for everyone else
GCBF_GHD const float* cond_source_state(int64_t src, int64_t a_node, const float* states, int ld, const float* s_moved) {
  return src == a_node ? s_moved : states + src * ld;
}

}  // namespace cond
}  // namespace gcbf
