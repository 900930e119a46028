// TEST INFRASTRUCTURE ONLY.  Sampling driver around the UNMODIFIED reference CPU path (ALGORITHM:GCNSAMPLESINGLE).
// Compiled against the reference headers where they lie (REF of oracle/Makefile; rule in oracle/sample.mk), nothing is
// copied into this repository, output goes to oracle/_ref/.  It builds the Graph, GNNDatum, FullyRepGraph and Sampler
// exactly as toolkits/GCN_CPU_SAMPLE.hpp:46-70,251-265 does, samples the FIRST train batch with the cfg's FANOUT and
// BATCH_SIZE (Sampler::reservoir_sample), and dumps, for every hop h of sampled_sgs, as raw little-endian binaries
// <outdir>/h<h>_<name>.bin:
//   dst, c_o, r_i (local source ids), src (first-appearance order), w (nts_norm_degree(src, dst) per edge),
//   X [n_src, F] = gen_x(src global id, f), Y = MiniBatchFuseOp(hop).forward(X),
//   G [n_dst, F] = gen_g(dst global id, f), dX = MiniBatchFuseOp(hop).backward(G).
// Run with NTS_THREADS=1: the reference backward accumulates into shared source rows from several threads.
//
// usage: nts_ref_sample_driver <cfg> <outdir> <F>
#include "core/neutronstar.hpp"
#include "core/ntsMiniBatchGraphOp.hpp"
#include <fstream>
#include <string>
#include <vector>

static std::string g_outdir;

template <class T> static void dump(const std::string &name, const T *p, size_t count) {
  std::ofstream f(g_outdir + "/" + name + ".bin", std::ios::binary);
  f.write(reinterpret_cast<const char *>(p), (std::streamsize)(count * sizeof(T)));
}
static void dump_tensor(const std::string &name, const NtsVar &t) {
  NtsVar c = t.contiguous();
  dump(name, c.data_ptr<float>(), (size_t)c.numel());
}

// the deterministic inputs of ref_driver.cpp, by global vertex id
static inline float gen_x(long v, long f, long F) { return sinf(0.37f * (float)((v * F + f) % 100003)); }
static inline float gen_g(long v, long f, long F) { return cosf(0.11f * (float)((v * F + f) % 100019)); }

int main(int argc, char **argv) {
  MPI_Instance mpi(&argc, &argv);
  if (argc < 4) {
    printf("usage: %s <cfg> <outdir> <F>\n", argv[0]);
    return 2;
  }
  g_outdir = argv[2];
  const int F = atoi(argv[3]);
  Graph<Empty> *graph = new Graph<Empty>();
  graph->config->readFromCfgFile(argv[1]);
  graph->replication_threshold = graph->config->repthreshold;
  graph->load_directed(graph->config->edge_file, graph->config->vertices);
  graph->generate_backward_structure();
  graph->init_gnnctx(graph->config->layer_string);
  graph->init_gnnctx_fanout(graph->config->fanout_string);
  graph->init_rtminfo();
  graph->rtminfo->with_weight = true;
  graph->rtminfo->with_cuda = false;
  GNNDatum *gnndatum = new GNNDatum(graph->gnnctx, graph);
  gnndatum->readFeature_Label_Mask(graph->config->feature_file, graph->config->label_file,
                                   graph->config->mask_file);
  FullyRepGraph *fully_rep_graph = new FullyRepGraph(graph);
  fully_rep_graph->GenerateAll();
  std::vector<VertexId> train_nids;
  for (int i = 0; i < graph->gnnctx->l_v_num; ++i)
    if (gnndatum->local_mask[i] == 0)
      train_nids.push_back(i);
  Sampler *sampler = new Sampler(fully_rep_graph, train_nids);
  const int hops = (int)graph->gnnctx->layer_size.size() - 1;
  sampler->reservoir_sample(hops, graph->config->batch_size, graph->gnnctx->fanout);
  SampledSubgraph *sg = sampler->get_one();

  long meta[4] = {hops, (long)graph->config->batch_size, F, (long)train_nids.size()};
  dump("meta", meta, 4);
  for (int h = 0; h < hops; h++) {
    sampCSC *b = sg->sampled_sgs[h];
    const std::string p = "h" + std::to_string(h) + "_";
    dump(p + "dst", b->dst().data(), b->dst().size());
    dump(p + "c_o", b->c_o().data(), b->c_o().size());
    dump(p + "r_i", b->r_i().data(), b->r_i().size());
    dump(p + "src", b->src().data(), b->src().size());
    std::vector<float> w;
    for (size_t d = 0; d < b->dst().size(); d++)
      for (VertexId e = b->c_o()[d]; e < b->c_o()[d + 1]; e++)
        w.push_back(nts::op::nts_norm_degree(graph, b->src()[b->r_i()[e]], b->dst()[d]));
    dump(p + "w", w.data(), w.size());
    const long n_src = (long)b->src().size(), n_dst = (long)b->dst().size();
    NtsVar X = torch::zeros({n_src, F}), G = torch::zeros({n_dst, F});
    for (long i = 0; i < n_src; i++)
      for (long f = 0; f < F; f++)
        X.data_ptr<float>()[i * F + f] = gen_x(b->src()[i], f, F);
    for (long i = 0; i < n_dst; i++)
      for (long f = 0; f < F; f++)
        G.data_ptr<float>()[i * F + f] = gen_g(b->dst()[i], f, F);
    nts::op::MiniBatchFuseOp op(sg, graph, h);
    NtsVar Y = op.forward(X);
    NtsVar dX = op.backward(G);
    dump_tensor(p + "X", X);
    dump_tensor(p + "Y", Y);
    dump_tensor(p + "G", G);
    dump_tensor(p + "dX", dX);
  }
  printf("nts_ref_sample_driver: %d hops, batch %d, F=%d\n", hops, (int)graph->config->batch_size, F);
  return 0;
}
