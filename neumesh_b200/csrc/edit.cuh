// Texture edit of a NeuMesh render (editing/texture_neumesh/texture_neumesh.py:81-121): per colour point, the main
// colour is blended with the colour networks of reference models over painted regions of the main mesh.  The handle
// (nmb_edit) and the kernels live in csrc/edit.cu; nmb_render_edit calls apply_edit after the main colour MLP.
#pragma once
#include "field.cuh"

namespace nmb {

// Scratch of one reference's pass over n colour points (SoA, stride n); references run one after another, so one
// set serves all of them.
struct EditScratch {
  int32_t* flag;      // [n]   point has painted weight
  int32_t* src;       // [n]   compacted list: colour point index of painted point j (ascending)
  int32_t* count;     // [1]   number of painted points
  float* ds;          // [n]
  int32_t* slot;      // [8][n] main-grid slots (the edit code table is in the same slot order)
  float* w_ref;       // [8][n] w_k m_k / (sum_k w_k m_k + 1e-8)
  float* nabla;       // [3][n] R_i nabla
  float* dirs;        // [n,3]  R_i view direction (row-major, FieldIn::dirs)
  float* a_paint;     // [n]
  float* a_rest;      // [n]
  float* rgb;         // [3][n] reference colour
  void* select_tmp;
  size_t select_bytes;
  int64_t total;      // floats
};

// carve the scratch for up to n colour points from `base` (nullptr: sizes only)
EditScratch edit_carve(void* base, int64_t n);

// true if any reference model's colour network takes nabla as an input
bool edit_needs_nabla(const nmb_edit* e);

// the main grid the edit's masks and codes are permuted to
const nmb_grid* edit_grid(const nmb_edit* e);

// false if that grid was updated (nmb_grid_update) after the edit's tables were permuted to its slot order
bool edit_fresh(const nmb_edit* e);

// Blend the references of `e` into rgb ([3][in.stride] SoA, the main colour of the n points described by `in`:
// ds, slot, w, nabla (nullable unless a reference takes nabla), dirs or rays_d / R).  Reads one count back per
// reference (synchronises the stream).
int apply_edit(const nmb_edit* e, const FieldIn& in, int64_t n, float* rgb, const EditScratch& s, cudaStream_t stream);

}  // namespace nmb
