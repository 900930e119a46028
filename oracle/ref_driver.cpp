// TEST INFRASTRUCTURE ONLY.  Op-level driver around the UNMODIFIED reference CPU
// path.  It is compiled against the reference headers where they lie (REF of oracle/Makefile)
// (nothing is copied into this repository) by oracle/Makefile, output goes to
// oracle/_ref/.  It loads an edge file exactly as toolkits/main.cpp:44-54 does,
// builds the PartitionedGraph exactly as toolkits/GAT_CPU_DIST.hpp:67-74 does,
// runs the reference's own CPU graph operators on deterministic inputs and
// dumps every integer artefact and every float result as raw little-endian
// binaries, one set per rank:   <outdir>/r<rank>_<name>.bin
//
// Modes (argv[3]):
//   dump   - artefacts + operator results (golden vectors; Cora-sized inputs)
//   time   - op-level timing of ForwardCPUfuseOp forward/backward (CPU baseline)
//   adam   - the reference's Parameter (core/NtsScheduler.hpp:639-791) driven exactly as toolkits/GCN.hpp:209-215
//            drives it (all_reduce_to_gradient -> learn..._Adam -> next) on deterministic W / gradients for <F>
//            steps; dumps W, M, V after every step (golden vectors of the fused Adam kernel)
//
// usage: nts_ref_driver <cfg> <outdir> <dump|time|adam> <F> [repeats]
#include "core/neutronstar.hpp"
#include <fstream>
#include <string>
#include <vector>

static std::string g_outdir;
static int g_rank = 0;

template <class T> static void dump(const std::string &name, const T *p, size_t count) {
  std::string path = g_outdir + "/r" + std::to_string(g_rank) + "_" + name + ".bin";
  std::ofstream f(path, std::ios::binary);
  f.write(reinterpret_cast<const char *>(p), (std::streamsize)(count * sizeof(T)));
}
static void dump_tensor(const std::string &name, const NtsVar &t) {
  NtsVar c = t.contiguous();
  dump(name, c.data_ptr<float>(), (size_t)c.numel());
}

// Deterministic inputs, a function of the GLOBAL index so that a P-rank run and
// the single-rank run see the same matrix.
static inline float gen_x(long v, long f, long F) { return sinf(0.37f * (float)((v * F + f) % 100003)); }
static inline float gen_g(long v, long f, long F) { return cosf(0.11f * (float)((v * F + f) % 100019)); }
static inline float gen_e(long key) { return sinf(0.77f * (float)(key % 100043)) * 2.0f; }

int main(int argc, char **argv) {
  MPI_Instance mpi(&argc, &argv);
  if (argc < 5) {
    printf("usage: %s <cfg> <outdir> <dump|time> <F> [repeats]\n", argv[0]);
    return 2;
  }
  g_outdir = argv[2];
  std::string mode = argv[3];
  int F = atoi(argv[4]);
  int repeats = argc > 5 ? atoi(argv[5]) : 3;

  if (mode == "adam") {
    const int steps = F, w = 37, h = 11;
    Parameter *P = new Parameter(w, h, 0.01f, 0.9f, 0.999f, 1e-9f, 0.0001f); // toolkits/GCN.hpp:96-119
    P->set_decay(0.97f, 4);                                                  // the reference stores both in `int`
    NtsVar W0 = torch::zeros({w, h});
    for (int i = 0; i < w * h; i++)
      W0.data_ptr<float>()[i] = 0.1f * sinf(0.3f * (float)i);
    P->W.set_data(W0.clone());
    dump_tensor("adam_W0", W0);
    std::vector<float> all_g, all_W, all_M, all_V;
    for (int s = 0; s < steps; s++) {
      NtsVar g = torch::zeros({w, h});
      for (int i = 0; i < w * h; i++)
        g.data_ptr<float>()[i] = 0.02f * cosf(0.05f * (float)(s * w * h + i)) + 0.001f * (float)(i % 7);
      all_g.insert(all_g.end(), g.data_ptr<float>(), g.data_ptr<float>() + w * h);
      P->all_reduce_to_gradient(g);
      P->learnC2C_with_decay_Adam();
      P->next();
      NtsVar Wc = P->W.detach().contiguous(), Mc = P->M.contiguous(), Vc = P->V.contiguous();
      all_W.insert(all_W.end(), Wc.data_ptr<float>(), Wc.data_ptr<float>() + w * h);
      all_M.insert(all_M.end(), Mc.data_ptr<float>(), Mc.data_ptr<float>() + w * h);
      all_V.insert(all_V.end(), Vc.data_ptr<float>(), Vc.data_ptr<float>() + w * h);
    }
    long meta[3] = {w, h, steps};
    dump("adam_meta", meta, 3);
    dump("adam_grads", all_g.data(), all_g.size());
    dump("adam_W", all_W.data(), all_W.size());
    dump("adam_M", all_M.data(), all_M.size());
    dump("adam_V", all_V.data(), all_V.size());
    return 0;
  }

  Graph<Empty> *graph = new Graph<Empty>();
  graph->config->readFromCfgFile(argv[1]);
  g_rank = graph->partition_id;
  graph->replication_threshold = graph->config->repthreshold;
  graph->load_directed(graph->config->edge_file, graph->config->vertices);
  graph->generate_backward_structure();

  VertexSubset *active = graph->alloc_vertex_subset();
  active->fill();
  graph->init_gnnctx(graph->config->layer_string);
  graph->init_rtminfo();
  graph->rtminfo->process_local = graph->config->process_local;
  graph->rtminfo->reduce_comm = graph->config->process_local;
  graph->rtminfo->copy_data = false;
  graph->rtminfo->process_overlap = graph->config->overlap;
  graph->rtminfo->with_weight = true;
  graph->rtminfo->with_cuda = false;
  graph->rtminfo->lock_free = graph->config->lock_free;

  PartitionedGraph *pg = new PartitionedGraph(graph, active);
  pg->GenerateAll(
      [&](VertexId s, VertexId d) { return nts::op::nts_norm_degree(graph, s, d); },
      CPU_T, true);
  graph->init_communicatior();

  const long V = graph->vertices;
  const int P = graph->partitions;
  const long v0 = graph->partition_offset[g_rank];
  const long Vp = graph->owned_vertices;
  const long Ep = pg->owned_edges;
  const long M = pg->owned_mirrors;

  NtsVar X = torch::zeros({Vp, F});
  NtsVar G = torch::zeros({Vp, F});
  {
    float *x = X.data_ptr<float>();
    float *g = G.data_ptr<float>();
    for (long v = 0; v < Vp; v++)
      for (long f = 0; f < F; f++) {
        x[v * F + f] = gen_x(v0 + v, f, F);
        g[v * F + f] = gen_g(v0 + v, f, F);
      }
  }

  if (mode == "time") {
    nts::op::ForwardCPUfuseOp op(pg, active);
    double best_f = 1e30, best_b = 1e30;
    for (int it = 0; it < repeats + 1; it++) {
      double t0 = get_time();
      NtsVar Y = op.forward(X);
      double t1 = get_time();
      NtsVar dX = op.backward(G);
      double t2 = get_time();
      if (it > 0 || repeats == 0) { // first call grows the message buffers
        best_f = std::min(best_f, t1 - t0);
        best_b = std::min(best_b, t2 - t1);
      }
    }
    if (g_rank == 0) {
      printf("{\"ref_cpu\": true, \"threads\": %d, \"V\": %ld, \"E\": %ld, \"F\": %d, "
             "\"forward_s\": %.6f, \"backward_s\": %.6f}\n",
             graph->threads, V, (long)graph->edges, F, best_f, best_b);
      fflush(stdout);
    }
    return 0;
  }

  // ---- integer artefacts ------------------------------------------------------
  long meta[8] = {V, (long)graph->edges, P, g_rank, Vp, Ep, M, F};
  dump("meta", meta, 8);
  dump("partition_offset", graph->partition_offset, (size_t)P + 1);
  dump("out_degree", graph->out_degree_for_backward, (size_t)V);
  dump("in_degree", graph->in_degree_for_backward, (size_t)V);
  for (int i = 0; i < P; i++) {
    CSC_segment_pinned *c = pg->graph_chunks[i];
    std::string tag = "chunk" + std::to_string(i) + "_";
    int cm[8] = {c->edge_size,    c->batch_size_forward, c->batch_size_backward, c->src_range[0],
                 c->src_range[1], c->dst_range[0],       c->dst_range[1],        0};
    dump(tag + "meta", cm, 8);
    dump(tag + "column_offset", c->column_offset, (size_t)c->batch_size_forward + 1);
    dump(tag + "row_indices", c->row_indices, (size_t)c->edge_size);
    dump(tag + "edge_weight_forward", c->edge_weight_forward, (size_t)c->edge_size);
    dump(tag + "row_offset", c->row_offset, (size_t)c->batch_size_backward + 1);
    dump(tag + "column_indices", c->column_indices, (size_t)c->edge_size);
    dump(tag + "edge_weight_backward", c->edge_weight_backward, (size_t)c->edge_size);
    // source_active: which vertices of partition i have an edge into this rank
    std::vector<unsigned char> act((size_t)c->batch_size_backward);
    for (int v = 0; v < c->batch_size_backward; v++)
      act[v] = c->source_active->get_bit(v) ? 1 : 0;
    dump(tag + "source_active", act.data(), act.size());
    // hasMirrorAtPartition[i]: which LOCAL vertices partition i needs
    std::vector<unsigned char> mir((size_t)Vp);
    for (long v = 0; v < Vp; v++)
      mir[v] = pg->hasMirrorAtPartition[i]->get_bit(v) ? 1 : 0;
    dump(tag + "has_mirror_at", mir.data(), mir.size());
  }
  dump("mirror_index", pg->MirrorIndex, (size_t)V + 1);
  dump("whole_column_offset", pg->column_offset, (size_t)Vp + 1);
  dump("whole_row_indices", pg->row_indices, (size_t)Ep);
  dump("whole_compressed_row_offset", pg->compressed_row_offset, (size_t)M + 1);
  dump("whole_column_indices", pg->column_indices, (size_t)Ep);

  // ---- fused GCN aggregation (core/ntsCPUFusedGraphOp.hpp) -----------------------
  dump_tensor("X", X);
  dump_tensor("G", G);
  {
    nts::op::ForwardCPUfuseOp op(pg, active);
    NtsVar Y = op.forward(X);
    NtsVar dX = op.backward(G);
    dump_tensor("gcn_Y", Y);
    dump_tensor("gcn_dX", dX);
  }

  // ---- distributed edge operators (core/ntsDistCPUGraphOp.hpp) ------------------
  NtsVar mirror;
  {
    nts::op::DistGetDepNbrOp op(pg, active);
    mirror = op.forward(X);
    dump_tensor("dep_mirror", mirror);
    NtsVar Gm = torch::zeros({M, F});
    float *gm = Gm.data_ptr<float>();
    // mirror slot m belongs to the global source s with MirrorIndex[s]==m
    for (long s = 0; s < V; s++)
      if (pg->MirrorIndex[s + 1] != pg->MirrorIndex[s])
        for (long f = 0; f < F; f++)
          gm[(long)pg->MirrorIndex[s] * F + f] = gen_g(s, f, F) * (1.0f + 0.125f * g_rank);
    dump_tensor("dep_Gm", Gm);
    NtsVar dXm = op.backward(Gm);
    dump_tensor("dep_dX", dXm);
  }
  NtsVar Ge = torch::zeros({Ep, F});
  {
    float *ge = Ge.data_ptr<float>();
    for (long e = 0; e < Ep; e++)
      for (long f = 0; f < F; f++)
        ge[e * F + f] = gen_e((long)pg->row_indices[e] * 131 + e * 7 + f + 1009L * g_rank);
    dump_tensor("Ge", Ge);
  }
  {
    nts::op::DistScatterSrc op(pg, active);
    NtsVar msg = op.forward(mirror);
    dump_tensor("scatter_src_msg", msg);
    NtsVar dm = op.backward(Ge);
    dump_tensor("scatter_src_dmirror", dm);
  }
  {
    nts::op::DistScatterDst op(pg, active);
    NtsVar msg = op.forward(X);
    dump_tensor("scatter_dst_msg", msg);
    NtsVar dx = op.backward(Ge);
    dump_tensor("scatter_dst_dX", dx);
  }
  {
    nts::op::DistAggregateDst op(pg, active);
    NtsVar y = op.forward(Ge);
    dump_tensor("aggregate_dst_Y", y);
    NtsVar dmsg = op.backward(G);
    dump_tensor("aggregate_dst_dmsg", dmsg);
  }
  NtsVar att;
  {
    NtsVar m = torch::zeros({Ep, 1});
    NtsVar ga = torch::zeros({Ep, 1});
    float *mp = m.data_ptr<float>();
    float *gp = ga.data_ptr<float>();
    for (long e = 0; e < Ep; e++) {
      mp[e] = gen_e((long)pg->row_indices[e] * 17 + e * 3 + 5 + 31L * g_rank);
      gp[e] = gen_e((long)pg->row_indices[e] * 29 + e * 11 + 7 + 37L * g_rank) * 0.5f;
    }
    dump_tensor("softmax_in", m);
    dump_tensor("softmax_gout", ga);
    nts::op::DistEdgeSoftMax op(pg, active);
    att = op.forward(m);
    dump_tensor("softmax_out", att);
    NtsVar gin = op.backward(ga);
    dump_tensor("softmax_gin", gin);
  }
  {
    nts::op::DistAggregateDstFuseWeight op(pg, active);
    NtsVar y = op.forward(mirror, att);
    dump_tensor("fuse_Y", y);
    NtsVar dm = op.backward(G);
    dump_tensor("fuse_dmirror", dm);
    NtsVar dw = op.get_additional_grad();
    dump_tensor("fuse_dweight", dw);
  }
  MPI_Barrier(MPI_COMM_WORLD);
  if (g_rank == 0)
    printf("nts_ref_driver: dumped P=%d V=%ld E=%ld F=%d\n", P, V, (long)graph->edges, F);
  return 0;
}
