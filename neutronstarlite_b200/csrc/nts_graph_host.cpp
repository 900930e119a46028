// Host-side graph preparation behind the C ABI (no device code): the layout contract of the reference's
// loader / partitioner / chunk builder, restated so a caller can hand this library a packed binary edge list
// ({u32 src, u32 dst}, dep/gemini/type.hpp:100-106) and get the exact arrays the kernels consume.
//
//   degrees            core/graph.hpp:1160-1181,1373,1414-1417 (+ clamp :4396-4401)
//   partition offsets  core/graph.hpp:1185-1211  (alpha = 12*(P+1) :408, PAGESIZE = 1024 rounding :1203)
//   edge weight        core/ntsBaseOp.hpp:194-197 (nts_norm_degree)
//   chunks             core/PartitionedGraph.hpp:324-420 (CSC + CSR per source partition, source_active :397)
//   MirrorIndex        core/PartitionedGraph.hpp:295-305
//
// Orders are canonical: CSC = (dst, src) ascending (what the reference produces), CSR = (src, dst) ascending
// (the reference's order inside a source row depends on thread timing in load_directed; any order is valid).
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "nts_b200.h"

namespace {

const uint32_t kPageSize = 1u << 10; // dep/gemini/constants.hpp

inline float norm_degree(uint32_t out_deg_src, uint32_t in_deg_dst) {
  return 1 / ((float)std::sqrt((double)out_deg_src) * (float)std::sqrt((double)in_deg_dst));
}

} // namespace

namespace nts {

// core/graph.hpp:1185-1211 over the raw (un-clamped) out-degree; shared with the device builder (nts_graph_build.cu)
int partition_offsets_from_out_degree(const uint32_t *out_degree, uint64_t n_edges, nts_vid_t V, int P,
                                      nts_vid_t *partition_offset) {
  const uint64_t alpha = 12ull * (uint64_t)(P + 1);
  uint64_t remained = n_edges + (uint64_t)V * alpha;
  partition_offset[0] = 0;
  for (int i = 0; i < P; i++) {
    const uint64_t parts_left = (uint64_t)(P - i);
    const uint64_t expected = remained / parts_left;
    if (parts_left == 1) {
      partition_offset[i + 1] = V;
    } else {
      uint64_t got = 0;
      nts_vid_t cut = partition_offset[i]; // (the reference leaves this unset if the sum never exceeds)
      for (nts_vid_t v = partition_offset[i]; v < V; v++) {
        got += out_degree[v] + alpha;
        if (got > expected) {
          cut = v;
          break;
        }
      }
      partition_offset[i + 1] = cut / kPageSize * kPageSize;
    }
    for (nts_vid_t v = partition_offset[i]; v < partition_offset[i + 1]; v++)
      remained -= out_degree[v] + alpha;
  }
  return partition_offset[P] == V ? 0 : -1;
}

} // namespace nts

extern "C" {

int nts_host_degrees(const nts_vid_t *edges, uint64_t n_edges, nts_vid_t V, nts_vid_t *out_degree,
                     nts_vid_t *in_degree) {
  if (!edges || !out_degree || !in_degree)
    return -1;
  memset(out_degree, 0, sizeof(nts_vid_t) * (size_t)V);
  memset(in_degree, 0, sizeof(nts_vid_t) * (size_t)V);
  for (uint64_t e = 0; e < n_edges; e++) {
    nts_vid_t s = edges[2 * e], d = edges[2 * e + 1];
    if (s >= V || d >= V)
      return -1;
    out_degree[s]++;
    in_degree[d]++;
  }
  for (nts_vid_t v = 0; v < V; v++) {
    if (out_degree[v] < 1)
      out_degree[v] = 1;
    if (in_degree[v] < 1)
      in_degree[v] = 1;
  }
  return 0;
}

int nts_host_partition_offsets(const nts_vid_t *edges, uint64_t n_edges, nts_vid_t V, int P,
                               nts_vid_t *partition_offset) {
  if (!edges || !partition_offset || P < 1)
    return -1;
  std::vector<uint32_t> out_degree((size_t)V, 0); // raw (un-clamped) out degree at this point of the loader
  for (uint64_t e = 0; e < n_edges; e++) {
    if (edges[2 * e] >= V)
      return -1;
    out_degree[edges[2 * e]]++;
  }
  return nts::partition_offsets_from_out_degree(out_degree.data(), n_edges, V, P, partition_offset);
}

int nts_host_chunk_edge_counts(const nts_vid_t *edges, uint64_t n_edges, const nts_vid_t *po, int P, int rank,
                               uint64_t *counts) {
  if (!edges || !po || !counts || rank < 0 || rank >= P)
    return -1;
  for (int i = 0; i < P; i++)
    counts[i] = 0;
  const nts_vid_t v0 = po[rank], v1 = po[rank + 1];
  for (uint64_t e = 0; e < n_edges; e++) {
    nts_vid_t s = edges[2 * e], d = edges[2 * e + 1];
    if (d < v0 || d >= v1)
      continue;
    int lo = 0, hi = P; // partition of s: po[lo] <= s < po[lo+1]; empty partitions are skipped naturally
    while (hi - lo > 1) {
      int mid = (lo + hi) / 2;
      if (po[mid] <= s)
        lo = mid;
      else
        hi = mid;
    }
    counts[lo]++;
  }
  return 0;
}

int nts_host_build_chunk(const nts_vid_t *edges, uint64_t n_edges, nts_vid_t V, const nts_vid_t *po, int P,
                         int rank, int src_partition, const nts_vid_t *out_degree, const nts_vid_t *in_degree,
                         nts_vid_t *column_offset, nts_vid_t *row_indices, float *w_fwd, nts_vid_t *row_offset,
                         nts_vid_t *column_indices, float *w_bwd, unsigned char *source_active) {
  if (!edges || !po || !out_degree || !in_degree || !column_offset || !row_offset)
    return -1;
  if (rank < 0 || rank >= P || src_partition < 0 || src_partition >= P)
    return -1;
  (void)V;
  const nts_vid_t v0 = po[rank], v1 = po[rank + 1];
  const nts_vid_t s0 = po[src_partition], s1 = po[src_partition + 1];
  const size_t Vp = v1 - v0, Vi = s1 - s0;
  // select
  std::vector<uint64_t> sel;
  for (uint64_t e = 0; e < n_edges; e++) {
    nts_vid_t s = edges[2 * e], d = edges[2 * e + 1];
    if (d >= v0 && d < v1 && s >= s0 && s < s1)
      sel.push_back(e);
  }
  const size_t Ei = sel.size();
  if (Ei >= 0xffffffffull)
    return -1;
  // 1) stable bucket by source
  std::vector<uint32_t> cnt_src(Vi + 1, 0), cnt_dst(Vp + 1, 0);
  for (size_t k = 0; k < Ei; k++) {
    cnt_src[edges[2 * sel[k]] - s0 + 1]++;
    cnt_dst[edges[2 * sel[k] + 1] - v0 + 1]++;
  }
  for (size_t i = 0; i < Vi; i++)
    cnt_src[i + 1] += cnt_src[i];
  for (size_t i = 0; i < Vp; i++)
    cnt_dst[i + 1] += cnt_dst[i];
  memcpy(row_offset, cnt_src.data(), sizeof(uint32_t) * (Vi + 1));
  memcpy(column_offset, cnt_dst.data(), sizeof(uint32_t) * (Vp + 1));
  if (source_active) {
    for (size_t i = 0; i < Vi; i++)
      source_active[i] = cnt_src[i + 1] > cnt_src[i] ? 1 : 0;
  }
  if (Ei == 0)
    return 0;
  if (!row_indices || !column_indices)
    return -1;
  std::vector<uint32_t> by_src_s(Ei), by_src_d(Ei);
  {
    std::vector<uint32_t> pos(cnt_src.begin(), cnt_src.end() - 1);
    for (size_t k = 0; k < Ei; k++) {
      uint32_t s = edges[2 * sel[k]], d = edges[2 * sel[k] + 1];
      uint32_t p = pos[s - s0]++;
      by_src_s[p] = s;
      by_src_d[p] = d;
    }
  }
  // 2) stable bucket of that by destination -> CSC with ascending source inside a destination
  {
    std::vector<uint32_t> pos(cnt_dst.begin(), cnt_dst.end() - 1);
    for (size_t k = 0; k < Ei; k++) {
      uint32_t s = by_src_s[k], d = by_src_d[k];
      uint32_t p = pos[d - v0]++;
      row_indices[p] = s;
      if (w_fwd)
        w_fwd[p] = norm_degree(out_degree[s], in_degree[d]);
    }
  }
  // 3) stable bucket of the CSC by source -> CSR with ascending destination inside a source
  {
    std::vector<uint32_t> pos(cnt_src.begin(), cnt_src.end() - 1);
    for (size_t d_local = 0; d_local < Vp; d_local++) {
      for (uint32_t k = column_offset[d_local]; k < column_offset[d_local + 1]; k++) {
        uint32_t s = row_indices[k];
        uint32_t p = pos[s - s0]++;
        column_indices[p] = (uint32_t)(v0 + d_local);
        if (w_bwd)
          w_bwd[p] = norm_degree(out_degree[s], in_degree[v0 + d_local]);
      }
    }
  }
  return 0;
}

int nts_host_mirror_index(const nts_vid_t *edges, uint64_t n_edges, nts_vid_t V, const nts_vid_t *po, int rank,
                          nts_vid_t *mirror_index, nts_vid_t *owned) {
  if (!edges || !po || !mirror_index)
    return -1;
  const nts_vid_t v0 = po[rank], v1 = po[rank + 1];
  memset(mirror_index, 0, sizeof(nts_vid_t) * ((size_t)V + 1));
  for (uint64_t e = 0; e < n_edges; e++) {
    nts_vid_t s = edges[2 * e], d = edges[2 * e + 1];
    if (d >= v0 && d < v1)
      mirror_index[(size_t)s + 1] = 1;
  }
  for (size_t v = 0; v < V; v++)
    mirror_index[v + 1] += mirror_index[v];
  if (owned)
    *owned = mirror_index[V];
  return 0;
}

} // extern "C"

// ---- feature / label / mask tables (SURVEY 8 f3) --------------------------------------------------------------------
// GNNDatum::readFeature_Label_Mask (core/ntsDataloador.hpp:156-221) reads three text tables with one istream each,
// record by record: "id f0 .. fF-1", "id label", "id train|val|eval|test"; the k-th record of the label and mask
// tables belongs to the k-th record of the feature table (they are consumed in lock step, whatever their id column
// says), rows whose id lies in [v_begin, v_end) land at id - v_begin.  Same contract here, but the files are read
// whole and the records parsed in parallel (strtof: correctly rounded like the istream extraction).  A packed binary
// table (float32 [V, F] row-major, the twin of the reference's packed binary edge file) is read with one pread of the
// owned rows.
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <string>
#include <vector>

namespace {

bool slurp(const char *path, std::string *out) {
  int fd = open(path, O_RDONLY);
  if (fd < 0)
    return false;
  struct stat st;
  if (fstat(fd, &st) != 0) {
    close(fd);
    return false;
  }
  out->resize((size_t)st.st_size);
  size_t done = 0;
  while (done < out->size()) {
    ssize_t n = pread(fd, &(*out)[done], out->size() - done, (off_t)done);
    if (n <= 0)
      break;
    done += (size_t)n;
  }
  close(fd);
  return done == out->size();
}

// start offset of every non-empty line
std::vector<size_t> line_starts(const std::string &s) {
  std::vector<size_t> v;
  size_t i = 0, n = s.size();
  while (i < n) {
    while (i < n && (s[i] == '\n' || s[i] == '\r' || s[i] == ' ' || s[i] == '\t'))
      i++;
    if (i >= n)
      break;
    v.push_back(i);
    while (i < n && s[i] != '\n')
      i++;
  }
  return v;
}

} // namespace

extern "C" {

int nts_host_read_feature_label_mask(const char *feature_path, const char *label_path, const char *mask_path,
                                     nts_vid_t feature_size, nts_vid_t v_begin, nts_vid_t v_end, float *features,
                                     int64_t *labels, int32_t *masks) {
  if (!feature_path || !features || v_end < v_begin)
    return -1;
  std::string ftr, lbl, msk;
  if (!slurp(feature_path, &ftr))
    return -2;
  if (label_path && labels && !slurp(label_path, &lbl))
    return -3;
  if (mask_path && masks && !slurp(mask_path, &msk))
    return -4;
  const std::vector<size_t> fl = line_starts(ftr), ll = line_starts(lbl), ml = line_starts(msk);
  const int64_t n = (int64_t)fl.size();
  int bad = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(| : bad)
  for (int64_t k = 0; k < n; k++) {
    const char *p = ftr.c_str() + fl[k];
    char *end = nullptr;
    const unsigned long id = strtoul(p, &end, 10);
    if (end == p) {
      bad |= 1;
      continue;
    }
    if (id < v_begin || id >= v_end)
      continue;
    float *row = features + (size_t)(id - v_begin) * feature_size;
    p = end;
    for (nts_vid_t f = 0; f < feature_size; f++) {
      row[f] = strtof(p, &end);
      if (end == p)
        bad |= 2; // fewer than feature_size values on the line
      p = end;
    }
    if (labels && (size_t)k < ll.size()) {
      const char *q = lbl.c_str() + ll[k];
      strtoul(q, &end, 10); // the id column is read and ignored, like the reference's `input_lbl >> la`
      labels[id - v_begin] = strtol(end, nullptr, 10);
    }
    if (masks && (size_t)k < ml.size()) {
      const char *q = msk.c_str() + ml[k];
      strtoul(q, &end, 10);
      while (*end == ' ' || *end == '\t')
        end++;
      int m = 3; // core/ntsDataloador.hpp:196-205
      if (!strncmp(end, "train", 5))
        m = 0;
      else if (!strncmp(end, "eval", 4) || !strncmp(end, "val", 3))
        m = 1;
      else if (!strncmp(end, "test", 4))
        m = 2;
      masks[id - v_begin] = m;
    }
  }
  return bad ? -5 : 0;
}

// rows [v_begin, v_end) of a packed float32 [V, feature_size] table
int nts_host_read_feature_binary(const char *path, nts_vid_t feature_size, nts_vid_t v_begin, nts_vid_t v_end,
                                 float *features) {
  if (!path || !features || v_end < v_begin)
    return -1;
  int fd = open(path, O_RDONLY);
  if (fd < 0)
    return -2;
  const size_t row = (size_t)feature_size * sizeof(float);
  size_t want = (size_t)(v_end - v_begin) * row, done = 0;
  const off_t base = (off_t)((size_t)v_begin * row);
  char *dst = reinterpret_cast<char *>(features);
  while (done < want) {
    ssize_t n = pread(fd, dst + done, want - done, base + (off_t)done);
    if (n <= 0)
      break;
    done += (size_t)n;
  }
  close(fd);
  return done == want ? 0 : -3;
}

} // extern "C"
