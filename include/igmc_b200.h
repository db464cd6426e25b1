/* igmc_b200 — C-ABI of the H100-native IGMC hot path (libigmc_b200.so).
 *
 * The reference (muhanzhang/IGMC) has no FFI: its boundary is the Python API that Main.py
 * star-imports (Main.py:11-15).  The host side in igmc_b200/{util_functions,models,train_eval}.py
 * mirrors that API and calls ONLY the entry points below (via ctypes; INTEGRATION.md shows the
 * binding).  Every pointer is a DEVICE pointer owned by the caller (torch tensors), every call is
 * asynchronous on `stream` (a cudaStream_t passed as void*), returns 0 on success, a negative
 * value for argument errors, or 1000+cudaError for launch failures.  Data-dependent failures
 * (capacity overflow, malformed batch) are reported through the device-side error word `err`
 * (see IGMC_ERR_* in csrc/common.cuh) which the host checks at its next synchronisation point.
 *
 * Each entry point cites the reference code it replaces.
 */
#ifndef IGMC_B200_H
#define IGMC_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define IGMC_MAX_LAYERS 8
#define IGMC_HIDDEN 32      /* latent_dim entries are hard-coded to 32 in Main.py:391 */
#define IGMC_MAX_BASES 4    /* num_bases=4 in Main.py:394 (IGMC's default is 2) */
#define IGMC_LIN1_OUT 128   /* models.py:185 */
#define IGMC_MAX_HOP 3      /* --hop (Main.py:88, default 1); node features are one-hot of width 2h+2 */

/* Device-resident rating matrix.  Replaces SparseRowIndexer / SparseColIndexer
 * (util_functions.py:20-66): flat CSR + CSC, int32 indices, uint8 rating label (= stored value-1). */
typedef struct {
  const int32_t* row_ptr;   /* [num_users+1] */
  const int32_t* col_idx;   /* [nnz] ascending within a row */
  const uint8_t* rating;    /* [nnz] rating label 0..R-1 (the extractors flag IGMC_ERR_LABEL on a label >= R) */
  const int32_t* col_ptr;   /* [num_items+1] */
  const int32_t* row_idx;   /* [nnz] ascending within a column */
  int32_t num_users, num_items;
} igmc_csr_t;

/* Where graph g of a batch takes its (user, item, label) from.  Replaces the `links`/`labels`
 * members of MyDynamicDataset (util_functions.py:119-133) + DataLoader index sampling. */
typedef struct {
  const int64_t* idx;          /* [B] indices into links_*; NULL -> graph g uses entry g */
  const int32_t* links_u;      /* dataset-resident pairs */
  const int32_t* links_v;
  const int32_t* links_label;  /* rating label of the pair (y = class_values[label]); may be NULL */
  const int64_t* pair_id;      /* [B] sampling-stream id per graph; NULL -> idx[g] (or g) */
} igmc_pairs_t;

/* Scratch of igmc_extract_batch (per-graph node lists and counts). */
typedef struct {
  int32_t* nodes_u;  /* [B*cap] global user ids, target first then ascending */
  int32_t* nodes_v;  /* [B*cap] global item ids */
  int32_t* n_u;      /* [B] */
  int32_t* n_v;      /* [B] */
  int32_t* row_cnt;  /* [B*cap] */
  int32_t* m_cnt;    /* [B] undirected edges per graph */
  int32_t* col_cnt;  /* [B*cap] matches per item column */
  int32_t* hop_off;  /* [B*2*(IGMC_MAX_HOP+1)] nodes within distance d per side (users then items); needed for h > 1 */
  int32_t* sync;     /* [B+1] zero-initialised flags of the one-launch h = 1 path (re-armed by the kernel); NULL
                      * selects the generic two-launch path */
} igmc_extract_ws_t;

/* The collated batch in the reference's layout (what construct_pyg_graph + Batch.from_data_list
 * produce, util_functions.py:280-297) plus graph offsets.  Buffers are capacity-sized; the true
 * sizes are counts[0]=N, counts[1]=E (directed). */
typedef struct {
  int32_t node_cap, edge_cap, feat_dim;
  float* x;             /* [node_cap*feat_dim] one-hot of node_label, may be NULL */
  uint8_t* node_label;  /* [node_cap] 0 target user, 1 target item, 2 user, 3 item (h=1) */
  int64_t* batch;       /* [node_cap] graph id per node */
  int32_t* node_gid;    /* [node_cap] global user/item id per node */
  int64_t* edge_index;  /* [2*edge_cap]: row 0 at 0, row 1 at edge_cap */
  int64_t* edge_type;   /* [edge_cap] */
  float* y;             /* [B] */
  int32_t* node_ptr;    /* [B+1] */
  int32_t* edge_ptr;    /* [B+1] directed-edge offsets */
  int32_t* graph_nu;    /* [B] number of user nodes of each graph */
  int32_t* counts;      /* [2] N, E */
  /* optional (all or none): the message-passing adjacency of igmc_adj_t (symmetric form), built in the
   * same pass so that igmc_batch_prepare is not needed for extracted batches; lists sorted by (type, neighbour) */
  int32_t* adj_in_ptr;  /* [node_cap+1] */
  uint32_t* adj_in;     /* [edge_cap] */
  int32_t* adj_eid;     /* [edge_cap] */
  uint64_t* adj_tmp;    /* [edge_cap] scratch */
} igmc_batch_out_t;

/* Enclosing-subgraph extraction + labelling + graph construction + collate for B pairs, h = 1..IGMC_MAX_HOP hops.
 * Replaces MyDynamicDataset.get -> subgraph_extraction_labeling -> construct_pyg_graph
 * (util_functions.py:138-145, 208-297) and PyG's Batch.from_data_list.  `max_nodes_per_hop` < 0
 * means None; `cap` bounds one side's node list over all hops.  `inj_*` (all or none NULL) inject per-graph
 * node lists [B*cap] (test hook: the reference's own random.sample draw; h = 1 only).  `seed_dev` (optional, device) overrides `seed` so that a
 * captured CUDA graph can be replayed with a fresh sampling stream every step.
 * `num_classes` = len(class_values), `max_row_deg` = the longest user row of G (0 = unknown): with W->sync set they
 * let h = 1 batches take the one-launch path (single balanced row scan, look-back offsets; same outputs bit for bit).
 * A stored rating label or a pair label outside 0..num_classes-1 sets IGMC_ERR_LABEL and is written as 0. */
int igmc_extract_batch(const igmc_csr_t* G, const igmc_pairs_t* P, int B, int h, int max_nodes_per_hop,
                       double sample_ratio, uint64_t seed, const uint64_t* seed_dev, int cap,
                       const int32_t* inj_nodes_u, const int32_t* inj_nodes_v,
                       const int32_t* inj_n_u, const int32_t* inj_n_v,
                       const igmc_extract_ws_t* W, const float* class_values, int num_classes, int max_row_deg,
                       const igmc_batch_out_t* O, int* err, void* stream);

/* The path igmc_extract_batch and igmc_extract_sessions take for these arguments, without a launch: the dynamic shared
 * memory of the one-launch h = 1 kernel when the batch takes it, 0 for the generic two-launch kernels, -3 when neither
 * fits (the item table or the h > 1 bitmaps exceed shared memory; the extraction then returns -3 too), -2 / -4 for a
 * cap / h out of range.  `fast` = W->sync != NULL, `adjacency` = O->adj_in_ptr != NULL, `edge_cap` = O->edge_cap. */
int igmc_extract_plan(int num_users, int num_items, int B, int h, int cap, int num_classes, int max_row_deg,
                      int edge_cap, int fast, int adjacency);

/* Device-resident store of pre-extracted subgraphs: the reference's static `MyDataset` keeps
 * `(data, slices)` = every graph's tensors concatenated WITHOUT node offsets plus per-graph boundaries
 * (util_functions.py:92,108-109; SURVEY A.5b).  Same content here, in compact types, plus the adjacency. */
typedef struct {
  const int32_t* node_off;    /* [G+1] */
  const int32_t* edge_off;    /* [G+1] directed edges */
  const uint8_t* node_label;  /* [sum n] */
  const int32_t* node_gid;    /* [sum n] */
  const int32_t* edge_src;    /* [sum e] graph-local node ids */
  const int32_t* edge_dst;    /* [sum e] */
  const uint8_t* edge_type;   /* [sum e] */
  const float* y;             /* [G] */
  const int32_t* graph_nu;    /* [G] */
  const int32_t* adj_ptr;     /* [sum n + G] per graph n+1 graph-local list offsets */
  const uint32_t* adj_in;     /* [sum e] */
  const int32_t* adj_eid;     /* [sum e] graph-local directed edge ids */
} igmc_store_t;

/* Mini-batch assembly from the store for graphs idx[0..B): what InMemoryDataset.get + Batch.from_data_list do
 * for the static dataset (train_eval.py:46-51): concat, node-offset edge_index, build `batch`; outputs are the
 * same buffers igmc_extract_batch fills (adjacency included, symmetric form).  One CTA per graph, no host sync. */
int igmc_assemble_batch(const igmc_store_t* S, const int64_t* idx, int B, const igmc_batch_out_t* O, int* err,
                        void* stream);

/* Graph offsets of a foreign (PyG-collated) batch: node_ptr from `batch`, edge_ptr from the graph
 * of each edge's source.  Replaces what Batch.from_data_list knows implicitly.  Sets IGMC_ERR_BAD_BATCH when a batch
 * id lies outside [0, B) or below the previous node's, or an edge's source lies outside [0, N) or in a graph before
 * the previous edge's; node_ptr and edge_ptr are then undefined (do not pass them to igmc_batch_prepare). */
int igmc_batch_ptrs(const int64_t* batch, const int64_t* edge_src, int N, int E, int B,
                    int32_t* node_ptr, int32_t* edge_ptr, int* err, void* stream);

/* Message-passing adjacency of a batch: per node the incoming (and outgoing) edge lists sorted by
 * (edge_type, neighbour), entries pack nbr_local | type<<16; *_eid holds the directed edge id used to
 * index dropout draws.  `symmetric` != 0 (extractor output: [u|v ; v|u]) aliases out-lists to in-lists.
 * This is the private structure the fused RGCN kernels consume instead of PyG's per-edge gather
 * (RGCNConv.propagate, third party; call site models.py:201). */
typedef struct {
  int32_t* in_ptr;    /* [node_cap+1] */
  uint32_t* in_adj;   /* [edge_cap] */
  int32_t* in_eid;    /* [edge_cap] */
  int32_t* out_ptr;   /* same three for outgoing edges; ignored when symmetric */
  uint32_t* out_adj;
  int32_t* out_eid;
  uint64_t* tmp;      /* [edge_cap] scratch */
  int32_t symmetric;
} igmc_adj_t;

/* One CTA per graph, with 2 (n_cap + 1) ints of shared memory: returns -3 when that exceeds 200 KB.  A graph of more
 * than min(n_cap, 65535) nodes sets IGMC_ERR_SMEM_NODES and gets no lists.  An edge with an endpoint outside its
 * source's graph, or a type outside 0..255, sets IGMC_ERR_BAD_BATCH and joins no list (the lists of that graph then
 * leave slots unwritten).  The entry point does not know the model's relation count: types in [R, 256) are the
 * caller's to refuse (Batch.from_arrays records the type range; the models raise before any launch). */
int igmc_batch_prepare(const int64_t* edge_index, int64_t edge_row_stride, const int64_t* edge_type,
                       const int32_t* node_ptr, const int32_t* edge_ptr, int B, int n_cap,
                       const igmc_adj_t* A, int* err, void* stream);

/* IGMC parameters: one flat fp32 buffer (also the NCCL gradient bucket layout).
 * state_dict names of the reference (models.py:182-185, train_eval.py:168-172):
 *   convs.{l}.att [R,NB] | convs.{l}.basis [NB,in,32] | convs.{l}.root [in,32] | convs.{l}.bias [32]
 *   lin1.weight [128, 2*32*L] | lin1.bias [128] | lin2.weight [1,128] | lin2.bias [1] */
typedef struct {
  int32_t num_layers, num_relations, num_bases, in_dim0;
  int32_t off_att[IGMC_MAX_LAYERS], off_basis[IGMC_MAX_LAYERS], off_root[IGMC_MAX_LAYERS],
      off_bias[IGMC_MAX_LAYERS];
  int32_t off_lin1_w, off_lin1_b, off_lin2_w, off_lin2_b;
  int32_t conv_param_count;  /* params before off_lin1_w */
  int32_t param_count;
  float multiply_by;
  int32_t readout;           /* 0: IGMC target-row readout inside igmc_forward/igmc_backward (models.py:203-215);
                              * 1: none - igmc_forward stops at concat_states, igmc_backward takes S.dstate =
                              *    d loss / d concat_states from an external readout (igmc_sortpool_*) */
  int32_t list_hint;         /* 0 = unknown, else the number of edge-list entries one CTA should be able to stage in
                              * shared memory (largest per-CTA list seen + margin): the cluster plans then give up
                              * staging rows (more, smaller chunks) until the list buffer holds that many - large
                              * subgraphs (ml_100k, 402 nodes) otherwise gather through global memory */
} igmc_model_t;

/* Dropout draws of one step.  edge_keep/hidden_keep (uint8, 1 = keep) inject explicit draws
 * (parity tests); otherwise counter-hash draws keyed by `seed` are used when p > 0. */
typedef struct {
  float adj_dropout;            /* models.py:193-198, 0 disables */
  float hidden_dropout;         /* 0.5 in training (models.py:212), 0 in eval */
  uint64_t seed;
  const uint64_t* seed_dev;     /* optional device word overriding `seed` (CUDA-graph replay) */
  const uint8_t* edge_keep;     /* [E] or NULL */
  const uint8_t* hidden_keep;   /* [B*128] or NULL */
} igmc_dropout_t;

/* Activations kept between forward and backward. */
typedef struct {
  float* states;    /* [node_cap * 32*L]  concat_states (models.py:203) */
  float* zsave;     /* training only, NULL in eval.  cluster plans: [node_cap * R*in0p] 1/deg-scaled relation-space
                     * aggregate of the one-hot input (layer 0 only, in0p = in_dim0 rounded up to 4; layers >= 1 take
                     * their weight gradients from the backward's own aggregate and need nothing saved);
                     * generic plan (cluster 0): [L * node_cap * NB*32] basis-space aggregates of every layer */
  float* inv_deg;   /* [node_cap] 1/max(kept in-degree,1) */
  float* feat;      /* [B * 2*32*L] target-user | target-item rows */
  float* hid;       /* [B * 128] relu(lin1) after dropout scaling */
  float* hid_gscale;/* [B * 128] d hid / d pre-activation */
  float* pred;      /* [B] */
  int32_t* target;  /* [B*2] batch-global index of the target user / item node */
  int32_t node_cap; /* row count of one zsave / dstate layer slab */
  float* dstate;    /* [node_cap * 32*L] d loss / d concat_states written by an external readout; read by
                     * igmc_backward when readout = 1, unused otherwise */
  const float* wprep; /* [L * 2 * 32*((R+1)*32+4)] per-step prepared weights (igmc_prep_weights), cluster plans only */
  long long* prof;    /* optional debug: [grid][64] clock64() stamps of the kernel phases (cluster plans), or NULL */
  int32_t* gate;      /* optional: every CTA of igmc_forward (cluster plans) adds 1 when it starts, see igmc_gate_wait */
  float* l2_scratch;  /* [2 * node_cap * 32] backward scratch of the L2 plan (d pre / d h of two layers), else unused */
  float* rel_inv_deg; /* NULL: PyG 1.4.2 RGCNConv, one mean over all kept in-edges of a node (1/deg(v), inv_deg).
                       * Non-NULL, [node_cap * R]: PyG >= 1.6 RGCNConv(aggr='mean'), one mean per relation -
                       * x'_v = x_v root + bias + sum_r 1/|N_r(v)| sum_{u in N_r(v)} x_u W_r.  igmc_forward fills
                       * rel_inv_deg[v*R + r] = 1/max(kept in-edges of type r at v, 1) and normalises with it;
                       * igmc_backward / igmc_forward_backward read it.  The forward and backward of one step must agree
                       * on the mode.  Every plan supports both; plans, shared memory and list images are the same. */
} igmc_saved_t;

/* Launch-order gate for work that should run BESIDE the forward kernel without taking SMs from it (the extraction of
 * the next batch on a second stream): a one-warp kernel that returns once `target` more CTAs (= the forward's grid
 * size: all of its one-per-SM clusters are resident) have counted in, or after `timeout_us`.  `gate` = two zero-
 * initialised int32 words (started-CTA count, expected total; never reset).  Enqueue it on the second stream in front
 * of the work to be held back; exactly ONE forward per gate - the one of the same step - must be given `gate` through
 * igmc_saved_t (other forwards pass NULL). */
int igmc_gate_wait(int32_t* gate, int target, int timeout_us, void* stream);

/* Pre-staged edge lists of one batch for the cluster plans (igmc_stage_lists): per (graph, cluster rank) the
 * compacted, kept (after this step's dropout_adj draws, models.py:193-198), pre-swizzled list entries of the rank's
 * own nodes plus the segment tables the gather hands out work from - everything the model kernels otherwise rebuild
 * in their prologues.  The kernels pull an image into shared memory with two bulk (TMA) copies.
 * One image per direction: forward = in-lists, backward = out-lists. */
typedef struct {
  int32_t* tab;       /* [B*cluster][tab_ints] header (entries, segments, staged, own nodes) + segment tables */
  uint32_t* ent;      /* [B*cluster][lcap] staged entries */
  float* inv_deg;     /* [node_cap] 1/max(kept in-degree,1); forward image only (NULL in the backward image) */
  int32_t tab_ints, lcap, chunk, cluster;   /* the consuming kernel's plan, see igmc_stage_plan */
} igmc_stage_t;

/* Shape of the image the forward (backward = 0) / backward (1) kernel of plan `cluster` expects for subgraphs of up
 * to n_cap nodes: fills tab_ints, lcap, chunk, cluster of *img (pointers untouched).  Negative if the plan does not
 * exist. */
int igmc_stage_plan(const igmc_model_t* M, int n_cap, int cluster, int backward, igmc_stage_t* img);

/* Build the images of a prepared batch: `fwd` always, `bwd` when training != 0 (may be NULL otherwise).  The dropout
 * descriptor must be the one the forward / backward of this step will be given (same seed).  Replaces, once per
 * batch and off the critical path, the list staging of igmc_forward / igmc_backward. */
int igmc_stage_lists(const igmc_model_t* M, const int32_t* node_ptr, const int32_t* edge_ptr, const igmc_adj_t* A,
                     int B, int n_cap, const igmc_dropout_t* D, int training, const igmc_stage_t* fwd,
                     const igmc_stage_t* bwd, int* err, void* stream);

/* W_r = sum_b att[r,b] basis[b] (and its transpose) for every layer, once per step, so that the
 * per-subgraph CTAs only copy them into shared memory.  Required before igmc_forward / igmc_backward with
 * cluster > 0 whenever the parameters changed (reference: the same product inside RGCNConv.message and the
 * ARR term, train_eval.py:169-172). */
int igmc_prep_weights(const igmc_model_t* M, const float* params, float* wprep, void* stream);

/* Kernel plan.  `cluster` = 0 selects the generic kernels (csrc/rgcn.cu: one 256-thread CTA per
 * subgraph, any num_relations <= 256); 1/2/4 select the relation-space kernels (csrc/rgcn_rs.cu,
 * num_relations <= 12) with that many CTAs (a thread-block cluster) per subgraph; IGMC_PLAN_L2(c), c = 1/2/4/8,
 * selects the L2 plan (csrc/rgcn_l2.cu): the generic plan's arithmetic on a cluster of c CTAs per subgraph with the
 * node features in global memory (L2) instead of shared memory, for subgraphs of up to 65 535 nodes and any
 * num_relations <= 256.  Returns the dynamic shared memory in bytes the chosen kernel needs for subgraphs of up to
 * n_cap nodes (for the L2 plan the same for every n_cap <= 65 535), or a negative value if the plan is not available
 * (too many relations / does not fit in 227 KB / n_cap > 65 535). */
#define IGMC_PLAN_L2_BASE 16
#define IGMC_PLAN_L2(c) (IGMC_PLAN_L2_BASE + (c))
#define IGMC_L2_MAX_NODES 65535
int igmc_model_plan(const igmc_model_t* M, int n_cap, int cluster, int backward);

/* IGMC.forward for a prepared batch (models.py:190-217): 4x (RGCNConv + tanh), concat, target-row
 * readout, lin1/relu/dropout/lin2.  Node features resident in shared memory for all layers.
 * If `y` != NULL also writes dpred[g] = d(mean squared error)/d(lin2 output) for the fused train step
 * (train_eval.py:162), with `loss_scale` = 1/(global number of graphs). */
int igmc_forward(const igmc_model_t* M, const float* params, const uint8_t* node_label,
                 const int32_t* node_ptr, const int32_t* edge_ptr, const igmc_adj_t* A, int B, int n_cap,
                 const igmc_dropout_t* D, int training, const igmc_saved_t* S, const float* y,
                 float loss_scale, float* dpred, float* sqerr, int cluster, const igmc_stage_t* stage, int* err,
                 void* stream);

/* Backward of igmc_forward given dpred [B] (gradient wrt the lin2 output).  Writes partial gradients of
 * the conv parameters, one row per CTA, and the readout factors dhid [B*128]; igmc_grad_reduce turns them into the
 * flat gradient.  Row layout: cluster 0 -> gpart[B][conv_param_count] in parameter layout; IGMC_PLAN_L2(c) ->
 * gpart[B*c][conv_param_count] in parameter layout (S.l2_scratch required); cluster 1..4 ->
 * gpart[B*cluster][igmc_raw_grad_count()] "raw" rows (per layer dW_r [R][in0p|32][32] | d root | d bias): the
 * (att, basis) chain rule is linear and is applied once to the sum by igmc_grad_reduce.  Must use the same `cluster`
 * as the forward that produced S.  `stage` (optional) = the backward image of igmc_stage_lists.
 * (autograd of models.py:190-217) */
int igmc_backward(const igmc_model_t* M, const float* params, const uint8_t* node_label,
                  const int32_t* node_ptr, const int32_t* edge_ptr, const igmc_adj_t* A, int B, int n_cap,
                  const igmc_dropout_t* D, const igmc_saved_t* S, const float* dpred,
                  float* gpart, float* dhid, int cluster, const igmc_stage_t* stage, int* err, void* stream);

/* igmc_forward (training, with the loss) immediately followed by igmc_backward for the same batch, as ONE launch: a
 * cluster goes from its subgraph's readout straight into its backward (d loss / d pred of a subgraph depends on that
 * subgraph's forward only).  Same arguments, same results bit for bit as the two calls; relation-space plans (1..4) with the IGMC
 * readout only.  What `loss = mse_loss(model(data), y); loss.backward()` spans in train_eval.py:160-175. */
int igmc_forward_backward(const igmc_model_t* M, const float* params, const uint8_t* node_label,
                          const int32_t* node_ptr, const int32_t* edge_ptr, const igmc_adj_t* A, int B, int n_cap,
                          const igmc_dropout_t* D, const igmc_saved_t* S, const float* y, float loss_scale,
                          float* dpred, float* sqerr, float* gpart, float* dhid, int cluster,
                          const igmc_stage_t* stage_fwd, const igmc_stage_t* stage_bwd, int* err, void* stream);

/* floats per raw gradient row of the cluster plans (see igmc_backward) */
int igmc_raw_grad_count(const igmc_model_t* M);

/* grad[p] = sum over gpart rows (conv; `raw_rows` != 0: raw rows of the cluster plans, chain rule
 * d basis[b] = sum_r att[r,b] dW_r, d att[r,b] = <dW_r, basis[b]> applied to the sum) ; lin1/lin2 gradients from
 * (dhid, feat, hid, dpred) ; + ARR * d/dW sum_l sum_r ||W_{r+1}-W_r||^2 (train_eval.py:167-174).  Also writes
 * loss_out[0] = sum_g sqerr[g]*loss_scale + ARR*reg  when loss_out != NULL.  `reg_ws` is a zero-initialised
 * scratch of IGMC_REDUCE_WS_FLOATS floats (partial dot products / regulariser values + int tickets, re-armed by the
 * kernel). */
#define IGMC_REDUCE_WS_FLOATS (IGMC_MAX_LAYERS * 32 * 64 + IGMC_MAX_LAYERS * 32 + 64)
int igmc_grad_reduce(const igmc_model_t* M, const float* params, int B, int gpart_rows, const float* gpart,
                     int raw_rows, const float* dhid, const float* feat, const float* hid, const float* dpred,
                     const float* sqerr, float loss_scale, float arr, float grad_scale,
                     float* grad, float* loss_out, float* reg_ws, void* stream);

/* torch.optim.Adam step (train_eval.py:54,177; lr/weight_decay semantics of torch 1.4 Adam, eps outside
 * the sqrt, no amsgrad) on the flat buffers.  `step_count` points at TWO device int64 words: the step
 * counter (incremented by the kernel) and a zero-initialised completion ticket;
 * grad is multiplied by grad_mul first (1/world after an NCCL sum); `lr_dev` (optional device float)
 * overrides `lr` so LR decay does not invalidate a captured graph.  Optional bookkeeping of the reference's
 * `total_loss += loss.item() * num_graphs` (train_eval.py:176) without a host sync: loss_acc[0] += loss_in[0] *
 * loss_weight. */
int igmc_adam_step(float* params, const float* grad, float* exp_avg, float* exp_avg_sq,
                   int64_t* step_count, int n, float lr, const float* lr_dev, float beta1, float beta2,
                   float eps, float weight_decay, float grad_mul, const float* loss_in, float* loss_acc,
                   float loss_weight, void* stream);

/* ---- data-parallel exchange + fused update (SURVEY 8e: the reference has no DP; world 1 reproduces its step) ----
 * Every rank owns one exchange allocation that all ranks of the node map (CUDA IPC): a double-buffered copy of its
 * gradient plus an array of arrival flags its peers write.  The collective library (NCCL / gloo) only carries the
 * 64-byte handles once at start-up. */
#define IGMC_MAX_RANKS 8
typedef struct {
  float* grad[IGMC_MAX_RANKS];    /* grad[r]: rank r's [2][stride] gradient buffers (r = rank: local memory) */
  int32_t* flag[IGMC_MAX_RANKS];  /* flag[r]: rank r's [IGMC_MAX_RANKS] arrival flags, flag[r][src] = last step src published */
  int64_t* state;                 /* local [4], zero-initialised: exchange step counter, then three int32 tickets */
  int32_t world, rank, stride, pad_;
} igmc_comm_t;

/* cudaMalloc + zero + IPC handle (64 bytes) of an exchange allocation / map a peer's / unmap / free. */
int igmc_comm_alloc(int64_t bytes, void** dev_ptr, unsigned char* handle64);
int igmc_comm_open(const unsigned char* handle64, void** dev_ptr);
int igmc_comm_close(void* peer_ptr);
int igmc_comm_free(void* dev_ptr);

/* igmc_grad_reduce (raw rows) -> all-reduce(SUM) of the flat gradient over the ranks of `comm` -> igmc_adam_step,
 * as ONE kernel: the gradient is assembled into this rank's exchange buffer, the ranks publish / await each other's
 * arrival flags, and every thread sums its elements straight out of the peers' memory (NVLink, fixed rank order ->
 * bit-identical parameters on all ranks) before applying Adam.  Replaces `loss.backward()`'s accumulation +
 * `optimizer.step()` (train_eval.py:175-177) and the ncclAllReduce a DDP port would put between them.
 * `grad_copy` (optional) receives the reduced gradient.  `loss_ring` (optional; `ring_size` a power of two): the
 * step's loss is also stored at loss_ring[step number % ring_size] - pass mapped pinned HOST memory and the host reads
 * every step's loss (`loss.item()`, train_eval.py:176) without a copy launch or a sync.  `wprep` (optional): after
 * the update (second grid barrier) the kernel also rebuilds the prepared weights of igmc_prep_weights from the NEW
 * parameters, so that the next step's forward needs no separate preparation launch.
 * IGMC readout only (readout = 0), cluster plans only.  Returns -21 when the grid (one block per layer input row plus
 * the readout parameters) is larger than the device runs at once: its grid barriers need every block resident. */
int igmc_reduce_update(const igmc_model_t* M, float* params, int B, int gpart_rows, const float* gpart,
                       const float* dhid, const float* feat, const float* hid, const float* dpred,
                       const float* sqerr, float loss_scale, float arr, const igmc_comm_t* comm,
                       float* exp_avg, float* exp_avg_sq, int64_t* step_count, float lr, const float* lr_dev,
                       float beta1, float beta2, float eps, float weight_decay, float grad_mul,
                       float* loss_out, float* loss_acc, float loss_weight, float* reg_ws, float* grad_copy,
                       float* loss_ring, int ring_size, float* wprep, void* stream);

/* The grid igmc_reduce_update launches for model M: `blocks` (computed without a device) and, when `resident` is not
 * NULL, the blocks of that kernel the current device runs at once.  igmc_reduce_update returns -21 when
 * blocks > resident; callers then take igmc_grad_reduce -> all-reduce -> igmc_adam_step instead. */
int igmc_reduce_update_grid(const igmc_model_t* M, int* blocks, int* resident);

/* ---- SortPooling + 1-D convolution readout of DGCNN_RS (models.py:123-167 over DGCNN.__init__ models.py:65-85) ----
 * Consumes the concat_states a readout=1 igmc_forward produced.  latent_dim = [32,...,32,1] is run by the conv
 * kernels as 32-wide layers whose unused output columns have zero weights, so a states row has `state_stride` =
 * 32*L floats of which the first `width` = sum(latent_dim) are real and the sort key is column width-1.
 * Parameters (same flat bucket, reference state_dict names):
 *   conv1d_params1.weight [c1,1,width] .bias [c1] | conv1d_params2.weight [c2,c1,kw2] .bias [c2] |
 *   lin1.weight [128, dense_dim] .bias [128] | lin2.weight [1,128] .bias [1],  dense_dim = c2 * (k/2 - kw2 + 1). */
typedef struct {
  int32_t k, width, state_stride;
  int32_t c1, c2, kw2;       /* 16, 32, 5 (models.py:75-79) */
  int32_t t1, t2, dense_dim; /* k/2 ; t1 - kw2 + 1 ; c2 * t2 */
  int32_t off_conv1_w, off_conv1_b, off_conv2_w, off_conv2_b, off_lin1_w, off_lin1_b, off_lin2_w, off_lin2_b;
  int32_t param_begin, param_end;   /* the readout parameters' range in the flat bucket */
} igmc_sortpool_t;

typedef struct {
  int32_t* rank;      /* [node_cap] position of every node in its graph's order (last channel descending, ties by index) */
  int32_t* perm;      /* [B*k] batch-global node at position t, -1 = padding (graph smaller than k) */
  float* act1;        /* [B*c1*k]  relu(conv1) */
  float* pool;        /* [B*c1*t1] maxpool */
  float* flat;        /* [B*dense_dim] relu(conv2), channel-major (x.view(len(x), -1), models.py:161) */
  float* hid;         /* [B*128] relu(lin1) after dropout scaling */
  float* hid_gscale;  /* [B*128] */
  float* pred;        /* [B] */
  float* dhid;        /* [B*128] backward */
  float* gpart;       /* [B * (c1*width + c1 + c2*c1*kw2 + c2)] per-graph partial gradients of the two Conv1d */
} igmc_sortpool_saved_t;

/* Dynamic shared memory (bytes) of the readout kernels for graphs of up to n_cap nodes, negative if the
 * description is inconsistent or does not fit in 227 KB. */
int igmc_sortpool_plan(const igmc_sortpool_t* P, int n_cap, int backward);

/* global_sort_pool (PyG 1.4.2, SURVEY A.4) -> Conv1d -> ReLU -> MaxPool1d(2,2) -> Conv1d -> ReLU -> flatten -> lin1 ->
 * ReLU -> Dropout(0.5) -> lin2 -> [:,0] (models.py:155-165), one CTA per graph.  With y != NULL also
 * dpred[g] = d(mean squared error)/d pred and sqerr[g]. */
int igmc_sortpool_forward(const igmc_sortpool_t* P, const float* params, const float* states,
                          const int32_t* node_ptr, int B, int n_cap, const igmc_dropout_t* D, int training,
                          const igmc_sortpool_saved_t* S, const float* y, float loss_scale, float* dpred,
                          float* sqerr, int* err, void* stream);

/* Backward of igmc_sortpool_forward: writes dstate [N * state_stride] (= d loss / d concat_states, zero for nodes
 * that were not pooled and for the padding columns) for igmc_backward, and the readout parameters' gradients
 * (times grad_scale) into grad[param_begin, param_end). */
int igmc_sortpool_backward(const igmc_sortpool_t* P, const float* params, const float* states,
                           const int32_t* node_ptr, int B, int n_cap, const igmc_sortpool_saved_t* S,
                           const float* dpred, float* dstate, float grad_scale, float* grad, int* err,
                           void* stream);

/* ---- inference: candidate pairs + streaming per-user top-k (csrc/recommend.cu) ----
 * Scores pairs that have no rating and ranks them per user - what a trained model is for.  The reference has no such
 * path (its train_eval.py:182-245 only reduces labelled predictions to an RMSE); a user of it would build a dataset of
 * every candidate pair and loop over it in Python.  Here the candidates of a batch are produced on the device and
 * handed to igmc_extract_batch as an igmc_pairs_t with idx = NULL, the eval forward scores them (K checkpoints: K
 * forwards on the same batch), and the scores are merged into the running per-user top-k lists or scattered to
 * their pair index.  Sampling stream of every pair: pair_id = u * num_items + v, whatever batch it falls into. */
#define IGMC_TOPK_MAX 256
typedef struct {
  const int32_t* users;     /* recommend: [num_query] query users; NULL selects explicit pairs (pair_u, pair_v) */
  const int32_t* cand;      /* recommend: [num_cand] ascending, unique candidate items; NULL = every item of G.  With
                             * per_user: every query user's own list (igmc_candidate_lists), j's at [user_off[j],
                             * user_off[j+1]) */
  const int32_t* pair_u;    /* explicit pairs: [num_pairs] user / item of pair i */
  const int32_t* pair_v;
  int64_t* user_off;        /* recommend: [num_query+1] exclusive prefix of the per-user candidate counts (the plan) */
  int64_t* rated_off;       /* recommend with cand and exclude_rated: [num_query+1] offsets into rated_pos (the plan) */
  int32_t* rated_pos;       /* recommend with cand and exclude_rated: [sum of the query users' degrees] ascending
                             * positions in cand of each user's rated items (|row(u) & cand| entries per user) */
  int64_t num_pairs;        /* candidate pairs in all (recommend: user_off[num_query], known once the plan ran) */
  int32_t num_query, num_cand, exclude_rated;
  int32_t per_user;         /* 0: cand is one list shared by every query user (or NULL); 1: cand holds per-user lists
                             * and user_off from igmc_candidate_lists (which replaces igmc_candidate_plan) */
} igmc_candidates_t;

/* Per query user the number of candidate items (cand or every item, minus the user's rated items when exclude_rated:
 * num_items - deg(u) without a list) and their exclusive prefix user_off; with a list and exclude_rated also rated_off /
 * rated_pos.  ONE single-CTA launch.  User ids outside G set IGMC_ERR_CANDIDATES (and count 0). */
int igmc_candidate_plan(const igmc_csr_t* G, const igmc_candidates_t* Cd, int* err, void* stream);

/* Per-user candidate lists: `rows` [num_query, width] int32 names query slot j's candidate items, -1 = an empty slot.
 * The plan of a per_user run: every row sorted ascending (segmented radix sort into the workspace), deduplicated,
 * without the user's rated items when exclude_rated, written compactly to `lists` ([num_query * width] capacity)
 * at [user_off[j], user_off[j+1]), and the exclusive prefix user_off [num_query+1] of the counts.  Ids outside
 * [-1, num_items) and user ids outside G set IGMC_ERR_CANDIDATES (the slot / the user counts nothing).  Afterwards
 * set Cd->cand = lists, Cd->per_user = 1 and Cd->num_pairs = user_off[num_query] for igmc_candidate_pairs.
 * num_query * width < 2^31 - 1. */
int igmc_candidate_lists_ws_bytes(int num_query, int width, int64_t* bytes);
int igmc_candidate_lists(const igmc_csr_t* G, const igmc_candidates_t* Cd, const int32_t* rows, int width,
                         int32_t* lists, void* ws, int64_t ws_bytes, int* err, void* stream);

/* The pairs of global candidate positions [*cursor, *cursor + B) (positions ordered by query slot, then item), then
 * *cursor += B: `cursor` is a device word, so a captured graph replays with no host input.  Writes links_u / links_v /
 * pair_id [B] for igmc_extract_batch (idx = NULL) and tag [B] = the query slot (recommend) or the pair index
 * (explicit pairs).  Positions past num_pairs (the tail batch) repeat the last pair with tag -1, so every batch has the
 * same size and kernel plan.  Candidate rank c of a user maps to list position c + t, t = the number of the user's
 * rated positions r_q with r_q - q <= c (binary search; without a list the rated positions are the row's col_idx). */
int igmc_candidate_pairs(const igmc_csr_t* G, const igmc_candidates_t* Cd, int64_t* cursor, int B,
                         int32_t* links_u, int32_t* links_v, int64_t* pair_id, int64_t* tag, int* err, void* stream);

/* Item-side runs (recommend_users: per query item its best candidate users) run the three candidate kernels above on the
 * transposed view of G: an igmc_csr_t with row_ptr = G.col_ptr, col_idx = G.row_idx, col_ptr = G.row_ptr, row_idx =
 * G.col_idx, num_users = G.num_items, num_items = G.num_users and rating = NULL (G's ratings are not in column order).
 * igmc_candidate_plan, igmc_candidate_lists and igmc_candidate_pairs read only row_ptr, col_idx, num_users and
 * num_items of the igmc_csr_t they are given and never read rating, so they take such a view as it is: the query slots
 * are items, the candidates users and a slot's rated entries its raters.  Their pairs come out as (item, user);
 * igmc_item_query_pairs, run after igmc_candidate_pairs on the same batch, swaps links_u / links_v back to (user, item)
 * and rewrites pair_id = u * num_items + v (int64; num_items = G's), the pair id predict_pairs samples the pair with.
 * tag is left as it is; the tail (tag -1, the last pair repeated) is swapped like every other slot.  An item id outside
 * [0, num_items) or a negative user id sets IGMC_ERR_CANDIDATES (the pair becomes (0, 0)). */
int igmc_item_query_pairs(int num_items, int B, int32_t* links_u, int32_t* links_v, int64_t* pair_id, int* err,
                          void* stream);

/* Streaming top-k: s = (preds[0][i] + ... + preds[K-1][i]) / K in fp32, summed in checkpoint order (preds row stride B),
 * then every contiguous run of equal tag (one query user's candidates in this batch; tag -1 = padding) is merged into
 * that user's running list top_score / top_item [*, k] (ranked: score descending, then item ascending; NaN after every
 * number; empty slots = item -1, initialised by the caller, last).  One CTA per run, no float atomics: the result does
 * not depend on where batch boundaries fall.  1 <= k <= IGMC_TOPK_MAX. */
int igmc_topk_merge(const float* preds, int K, int B, const int64_t* tag, const int32_t* items, int k,
                    float* top_score, int64_t* top_item, void* stream);

/* 1 when a top-k merge of batch size B with k kept entries can launch, else 0: 1 <= k <= IGMC_TOPK_MAX, B >= 1 and the
 * merge's shared memory, 16 + (k + B) * 12 bytes (a head word, then a running list and the batch as int64 ids and
 * fp32 keys), within the 227 KB a CTA may take: k + B <= 19 369.  igmc_topk_merge refuses what does not fit with -2,
 * igmc_influence_topk (whose merge needs no head) with -20: one limit for both. */
int igmc_topk_fits(int k, int B);

/* Explicit pairs: scores[tag[i]] = the same fp32 checkpoint mean for every i with tag[i] >= 0. */
int igmc_score_scatter(const float* preds, int K, int B, const int64_t* tag, float* scores, void* stream);

/* ---- explanation by occlusion (csrc/explain.cu) ----
 * Why a pair got its score: for every rating of the pair's enclosing subgraph, the score of that subgraph without the
 * rating (both directed edges dropped, nodes unchanged, no re-sampling).  The reference only draws subgraphs for a look
 * (visualize, train_eval.py:248-322); a user of it would rebuild the subgraph per rating and call the model in a Python
 * loop.  Here a base pass of explicit pairs (igmc_candidate_pairs, igmc_score_scatter) counts each subgraph's ratings,
 * and an occlusion pass scores position c = (pair q, rating j) for every c < T = offsets[P]: igmc_extract_batch
 * extracts pair q again (same pair id: the same subgraph), igmc_occlusion_mask drops rating j through the model
 * kernels' edge_keep (training-mode forward, adj_dropout = hidden_dropout = 0: dropout_adj with that draw,
 * train_eval.py:160 / models.py:193-198) and igmc_score_scatter stores the score at c. */

/* After the extraction of a base batch: num_edges[tag[i]] = (edge_ptr[i+1] - edge_ptr[i]) / 2, the undirected edges of
 * graph i, for every i with tag[i] >= 0. */
int igmc_explain_count(const int32_t* edge_ptr, const int64_t* tag, int B, int32_t* num_edges, void* stream);

/* offsets [num_pairs+1]: the exclusive int64 prefix of num_edges; offsets[num_pairs] = T.  One CTA. */
int igmc_explain_offsets(const int32_t* num_edges, int num_pairs, int64_t* offsets, void* stream);

/* The pairs of occlusion positions [*cursor, *cursor + B), then *cursor += B (the igmc_candidate_pairs of an occlusion
 * pass): position c belongs to pair q, the last q with offsets[q] <= c, and names its rating j = c - offsets[q].
 * Writes links_u / links_v / pair_id = u * num_items + v (as predict_pairs samples the pair) / tag = c / edge_j = j.
 * Positions past T repeat the last position with tag -1.  Pair ids outside G set IGMC_ERR_CANDIDATES. */
int igmc_occlusion_pairs(const igmc_csr_t* G, const int32_t* pair_u, const int32_t* pair_v, const int64_t* offsets,
                         int num_pairs, int64_t* cursor, int B, int32_t* links_u, int32_t* links_v, int64_t* pair_id,
                         int64_t* tag, int32_t* edge_j, int* err, void* stream);

/* For the batch O of B graphs extracted from igmc_occlusion_pairs' output: edge_keep [O->edge_ptr[B]] is 1 except, in
 * every graph with tag >= 0, the two directed copies of its rating j (edge_ptr[g] + j and edge_ptr[g] + E_g/2 + j in
 * the [u|v ; v|u] edge_index); and user / item / rating [T] at position tag = the rating's global user, global item
 * and label.  One CTA per graph.  j outside the graph's ratings (a subgraph unlike the base pass's) sets
 * IGMC_ERR_CANDIDATES and drops nothing. */
int igmc_occlusion_mask(const igmc_batch_out_t* O, int B, const int64_t* tag, const int32_t* edge_j,
                        uint8_t* edge_keep, int32_t* user, int32_t* item, int32_t* rating, int* err, void* stream);

/* delta[c] = occluded[c] - score[q] (fp32) for every position, then each pair's segment [offsets[q], offsets[q+1])
 * ordered by |delta| descending, NaN after every number, ties by j (a segmented radix sort on the 64-bit key
 * (~orderable(|delta|) << 32) | j).  m = 0: out_* [T] in that order; 1 <= m <= IGMC_TOPK_MAX: out_* [num_pairs, m],
 * the first m entries of each segment, padded with user / item / rating -1 and delta 0.  `ws`: at least
 * igmc_occlusion_order_ws_bytes bytes.  num_pairs, num_positions < 2^31 - 1.  score = NULL: delta[c] = occluded[c]
 * (the values are ordered as they are; igmc_edge_grad_scatter's gradients). */
int igmc_occlusion_order_ws_bytes(int num_pairs, int64_t num_positions, int64_t* bytes);
int igmc_occlusion_order(const float* score, const float* occluded, const int64_t* offsets, int num_pairs,
                         int64_t num_positions, const int32_t* user, const int32_t* item, const int32_t* rating,
                         int m, void* ws, int64_t ws_bytes, int32_t* out_user, int32_t* out_item, int32_t* out_rating,
                         float* out_delta, void* stream);

/* ---- attribution by the score's gradient per rating (csrc/rgcn_l2.cu, csrc/explain.cu) ----
 * Each rating e of a subgraph gets a weight m_e that multiplies the messages of both its directed edges in every layer;
 * the normalisers count the weights (deg(v) = sum of m over v's in-edges; PyG >= 1.6 layers: |N_r(v)| = sum over v's
 * in-edges of type r), so that m in {0,1} is the edge_keep mask and m = 1 the model.  grad_e = d score / d m_e at m = 1.
 * Per directed edge j -> v of type r at layer l the term is (s - mean of s over v's segment) / |segment|, s =
 * <h_{l-1}[j] W_r, d pre_l[v]>; the segment is v's in-list (its in-edges of type r for PyG >= 1.6).  A single-edge
 * segment contributes 0 at that layer. */

/* Per directed edge, its terms summed over the layers: edge_grad [edge_ptr[B]], for a batch whose forward (evaluation:
 * D without edge dropout or edge_keep, else -18) ran on the plan IGMC_PLAN_L2(c) = `cluster` (any other plan: -16).
 * Operands as igmc_backward's, without gpart / dhid; dpred [B] = d score / d lin2 output (M->multiply_by for IGMC).
 * With readout = 1, S.dstate is d score / d concat_states (igmc_sortpool_backward seeded with the same dpred).  S.zsave
 * is not read.  Each element has one writer and a fixed layer order: bit-identical across runs. */
int igmc_edge_grad(const igmc_model_t* M, const float* params, const uint8_t* node_label, const int32_t* node_ptr,
                   const int32_t* edge_ptr, const igmc_adj_t* A, int B, int n_cap, const igmc_dropout_t* D,
                   const igmc_saved_t* S, const float* dpred, float* edge_grad, int cluster, int* err, void* stream);

/* One CTA per graph i of the batch O with tag[i] = q >= 0 (igmc_candidate_pairs over explicit pairs): for every rating
 * j < E_i/2, out[offsets[q] + j] = edge_grad[e0 + j] + edge_grad[e0 + E_i/2 + j] (e0 = edge_ptr[i]), accumulated over
 * checkpoints: checkpoint k = 0 stores, k > 0 adds in k order, k = K - 1 divides by K.  At k = 0 also user / item /
 * rating [T] as igmc_occlusion_mask records them.  A graph whose rating count is not its base-pass count sets
 * IGMC_ERR_CANDIDATES. */
int igmc_edge_grad_scatter(const igmc_batch_out_t* O, int B, const int64_t* tag, const float* edge_grad,
                           const int64_t* offsets, int k, int K, float* out, int32_t* user, int32_t* item,
                           int32_t* rating, int* err, void* stream);

/* ---- node explanations (csrc/explain.cu) ----
 * The explanation and attribution passes above with a pair's non-target nodes as positions: position j of graph g is
 * its j-th node with node_label >= 2 in node order (N_g - 2 positions for an extracted subgraph; the two targets are
 * not explained).  Occlusion drops every rating incident to the node (both directed edges; nodes, labels and sampling
 * unchanged), so an IGMC node sends no message: the node removed.  DGCNN_RS still sorts the isolated node into its
 * SortPooling.  The gradient of a node is d score / d g_n at g = 1 for a gate g_n on the weight m_e of each of its
 * ratings: the sum of those ratings' igmc_edge_grad_scatter values. */

/* After the extraction of a base batch: num_nodes[tag[i]] = max(node_ptr[i+1] - node_ptr[i] - 2, 0) for every i with
 * tag[i] >= 0.  igmc_explain_offsets scans the counts and igmc_occlusion_pairs maps the positions unchanged (its
 * edge_j is the node position j). */
int igmc_explain_node_count(const int32_t* node_ptr, const int64_t* tag, int B, int32_t* num_nodes, void* stream);

/* For the batch O of B graphs extracted from igmc_occlusion_pairs' output: edge_keep [O->edge_ptr[B]] is 1 except, in
 * every graph with tag >= 0, 0 on each directed edge with node p as source or target (both copies of each rating of
 * p), p = the graph's node at position node_j; and node / label / ratings [T] at position tag = p's global id
 * (node_gid), its node_label and its number of ratings in the subgraph.  One CTA per graph.  A position outside the
 * graph's nodes sets IGMC_ERR_CANDIDATES, drops nothing and records nothing. */
int igmc_node_occlusion_mask(const igmc_batch_out_t* O, int B, const int64_t* tag, const int32_t* node_j,
                             uint8_t* edge_keep, int32_t* node, int32_t* label, int32_t* ratings, int* err,
                             void* stream);

/* One CTA per graph i of the batch O (adjacency required) with tag[i] = q >= 0: for the node n at position j,
 * out[offsets[q] + j] = the fp32 sum over n's in-list entries adj_in_ptr[n] .. adj_in_ptr[n+1] (one per rating of n)
 * in list order, the first entry's value taken as it is, each later one added, of the rating's value
 * edge_grad[a] + edge_grad[a + E_i/2] (a = the rating's user -> item edge, e0 <= a < e0 + E_i/2); +0 without
 * entries.  Accumulated over checkpoints as igmc_edge_grad_scatter does: k = 0 stores, k > 0 adds in k order,
 * k = K - 1 divides by K.  At k = 0 also node / label / ratings [T] as igmc_node_occlusion_mask records them (ratings =
 * the in-list length).  A graph whose node count is not its base-pass count sets IGMC_ERR_CANDIDATES and writes
 * nothing. */
int igmc_node_grad_scatter(const igmc_batch_out_t* O, int B, const int64_t* tag, const float* edge_grad,
                           const int64_t* offsets, int k, int K, float* out, int32_t* node, int32_t* label,
                           int32_t* ratings, int* err, void* stream);

/* ---- per-pair gradients and training-data influence (csrc/influence.cu) ----
 * TracIn-CP (Pruthi et al., NeurIPS 2020): influence(i, t) = sum_k eta_k <grad l_i(theta_k), grad q_t(theta_k)> over
 * checkpoints k, self_influence(i) = sum_k eta_k ||grad l_i(theta_k)||^2, with l_i = (f_i - y_i)^2 of ONE pair (no batch
 * mean, no ARR term) and q_t = l_t (labelled test pair) or f_t (the score).  A gradient is the flat parameter vector in
 * the model's layout.  The per-pair gradient of graph g comes from the same backward as a training step (dropout rates 0):
 * its conv block is the sum of g's own partial rows, its readout block the rank-1 factors dhid (x) feat and dpred * hid. */

/* floats of one pair's factor row: dhid [128] | feat [2*32*L] | hid [128] | dpred [1] */
int igmc_pair_factor_count(const igmc_model_t* M);

/* dpred[g] = d l / d lin2 output for the backward: 2 (pred[g] - y[tag[g]]) multiply_by with y (the loss seed, the
 * forward's own dpred at loss_scale 1), multiply_by without (the score seed), 0 where tag[g] < 0 (padding). */
int igmc_pair_seed(const float* pred, const float* y, const int64_t* tag, int B, float multiply_by, float* dpred,
                   void* stream);

/* Per-graph gradients of a batch whose backward left gpart (rows_per_graph rows per graph, graph-major; raw_rows != 0:
 * the raw rows of the cluster plans, chain rule applied per graph) and the readout factors.  Row of graph g: g, or
 * tag[g] when `scatter` (tag < 0: nothing written); padding graphs of an unscattered batch get zeros.  grad (optional):
 * the conv block, row stride conv_param_count, or (full != 0) the whole gradient, row stride param_count, lin1 / lin2
 * materialised from the factors.  fac (optional): the factor rows (igmc_pair_factor_count floats).  IGMC readout only
 * (readout = 1: -16); raw rows need num_relations <= 12. */
int igmc_pair_grad(const igmc_model_t* M, const float* params, int B, int rows_per_graph, const float* gpart,
                   int raw_rows, const float* dhid, const float* feat, const float* hid, const float* dpred,
                   const int64_t* tag, int scatter, float* grad, int full, float* fac, void* stream);

/* self_out[tag[g]] += eta * ||G_g||^2 for every graph with tag >= 0, from its conv row (stride conv_param_count) and
 * factor row; one CTA per graph, fixed order. */
int igmc_self_influence(const igmc_model_t* M, int B, const float* conv, const float* fac, const int64_t* tag,
                        float eta, float* self_out, void* stream);

/* S[b][t] (= first ? 0 : S[b][t]) + eta * <G_b, G_t> for B training rows (conv_b [B][conv_param_count], fac_b) against T
 * test rows (conv_t, fac_t).  Conv block: split-K FFMA over fixed chunks of 256 entries, the splits summed in a fixed
 * order; readout block: (dhid_b . dhid_t)(feat_b . feat_t + 1) + dpred_b dpred_t (hid_b . hid_t + 1).  No float atomics:
 * bit-identical across runs and batch sizes.  `ws`: igmc_influence_ws_bytes bytes. */
int igmc_influence_ws_bytes(const igmc_model_t* M, int B, int T, int64_t* bytes);
int igmc_influence_accum(const igmc_model_t* M, int B, int T, const float* conv_b, const float* fac_b,
                         const float* conv_t, const float* fac_t, float eta, int first, void* ws, int64_t ws_bytes,
                         float* S, void* stream);

/* Per test pair t (one CTA each): the batch's values S[b][t] with index tag[b] (tag < 0 skipped) merged into the
 * running proponents (value descending) and opponents (value ascending) [T][k]; ties by index ascending, NaN after
 * every number, empty slots (index -1, value -inf / +inf, initialised by the caller) last.  A strict total order: the
 * result does not depend on batch boundaries.  1 <= k <= IGMC_TOPK_MAX. */
int igmc_influence_topk(const float* S, int B, int T, const int64_t* tag, int k, float* pro_value,
                        int64_t* pro_index, float* con_value, int64_t* con_index, void* stream);

/* ---- candidate retrieval by bridge count (csrc/retrieve.cu) ----
 * For h = 1 the enclosing subgraph of an unrated pair (u, v) joins u's star and v's star only through the bridge edges
 * (u', i): u' != u rated v and i, u rated i.  Their number is
 *   paths[v] = sum over u' != u of |N(u) & N(u')| * [u' rated v]
 * (the 3-paths u - i - u' - v).  Per query user the m items with the most bridges: items [num_query, m] and paths
 * [num_query, m] int32, ordered by paths descending, then item ascending; items with no bridge are never returned and
 * the rest of a row is item -1 / paths 0.  exclude_rated drops the user's rated items.  One CTA per user: pass 1 pushes
 * w[u'] (integer atomics, sum over i in N(u) of deg(i)), pass 2 pulls paths[v] = sum over col(v) of w (nnz reads), a
 * radix select of the m-th count (ties at it in ascending item order) and a bitonic sort of the chosen keys.  The
 * histograms w [num_users] and paths [num_items] live in shared memory when they fit, else in a workspace row per CTA
 * of a fixed grid (igmc_corated_ws_bytes: 0 in the shared-memory regime).  Integer arithmetic only: bit-identical
 * across runs.  User ids outside G set IGMC_ERR_CANDIDATES (their row is padding).  1 <= m <= num_items. */
int igmc_corated_ws_bytes(int num_users, int num_items, int num_query, int m, int64_t* bytes);
int igmc_corated_items(const igmc_csr_t* G, const int32_t* users, int num_query, int m, int exclude_rated, void* ws,
                       int64_t ws_bytes, int32_t* items, int32_t* paths, int* err, void* stream);

/* The item side of the same count: per query item v the m users u with the largest
 *   C[u][v] = (B B^T B)[u][v] - deg(u) * B[u][v]      (B the 0/1 rating matrix)
 * which is exactly the paths[v] igmc_corated_items gives user u.  `T` is the transposed view of G (see
 * igmc_item_query_pairs; rating is not read).  One CTA per item: pass 1 pushes w[i] += 1 for every rater u' of v and
 * every item i of u' (i = v included: w[v] = deg(v)), pass 2 pulls paths[u] = sum over i in row(u) of w[i], minus
 * deg(u) when row(u) holds v; then igmc_corated_items' select and sort.  users [num_query, m] / paths [num_query, m]
 * int32: paths descending, then user ascending; users without a bridge are never returned, the rest of a row is user -1
 * / paths 0; exclude_rated drops the item's raters.  Workspace igmc_corated_ws_bytes(G->num_items, G->num_users,
 * num_query, m) (T's shape).  Integer arithmetic, one writer per output: bit-identical across runs.  Item ids outside G
 * set IGMC_ERR_CANDIDATES (their row is padding).  1 <= m <= G->num_users. */
int igmc_corated_users(const igmc_csr_t* T, const int32_t* items, int num_query, int m, int exclude_rated, void* ws,
                       int64_t ws_bytes, int32_t* users, int32_t* paths, int* err, void* stream);

/* ---- in-place update of the rating graph (csrc/graph_update.cu) ----
 * The reference can only change its rating matrix by rebuilding everything from a new scipy matrix.  Here a delta of D
 * entries (users[i], items[i], values[i]) is applied to the graph's own device arrays; value = rating label + 1 (1..256)
 * inserts the rating or overwrites it, 0 deletes it (absent: nothing happens); within one call the last occurrence of a
 * pair wins.  The graph's arrays are allocated at capacity (cap_users + 1 / cap_items + 1 pointers, cap_nnz entries);
 * G describes the current shape and `nnz` its current entry count.  Afterwards the arrays are byte-identical, up to the
 * new nnz and shape, to a graph built from the updated matrix (CSR columns and CSC rows ascending), and the five
 * pointers are unchanged.  Ids below the capacity grow the shape to cover every id of the call; the shape never
 * shrinks.  The update is two calls with one host synchronisation between them (reading the header). */
typedef struct {
  int64_t nnz;                     /* entries after the update */
  int64_t num_users, num_items;    /* shape after the update */
  int64_t max_row_deg, max_col_deg;
  int64_t inserted, changed, removed;   /* kept entries that insert / change a label / delete; the rest change nothing */
  int32_t status;                  /* 0, or IGMC_GRAPH_UPDATE_OVER_CAPACITY / _OVER_INT32: apply must not run */
  int32_t err;                     /* the error word as the plan left it (IGMC_ERR_GRAPH_UPDATE: invalid delta) */
} igmc_graph_update_header_t;
#define IGMC_GRAPH_UPDATE_OVER_CAPACITY 1   /* new nnz > cap_nnz */
#define IGMC_GRAPH_UPDATE_OVER_INT32 2      /* new nnz beyond int32 */

/* Bytes of the workspace plan and apply share for a delta of D entries at these capacities. */
int igmc_graph_update_ws_bytes(int D, int cap_users, int cap_items, int cap_nnz, int64_t* bytes);

/* Validate (ids in [0, cap), values 0..256, else IGMC_ERR_GRAPH_UPDATE in `err`), order and classify the delta and
 * compute the new row_ptr / col_ptr into the workspace and the header (device).  `shape_users` / `shape_items`: the
 * least shape the call asks for (0 = none).  Changes nothing in G. */
int igmc_graph_update_plan(const igmc_csr_t* G, int nnz, int cap_users, int cap_items, int cap_nnz,
                           const int32_t* users, const int32_t* items, const int32_t* values, int D,
                           int shape_users, int shape_items, void* ws, int64_t ws_bytes,
                           igmc_graph_update_header_t* header, int* err, void* stream);

/* Merge the planned delta into G's arrays, written THROUGH G's pointers (they must be the graph's writable buffers).
 * Same G, nnz, capacities, D and workspace as the plan; new_nnz / new_users / new_items from its header, which must
 * report status 0 and err 0. */
int igmc_graph_update_apply(const igmc_csr_t* G, int nnz, int cap_users, int cap_items, int cap_nnz, int D,
                            void* ws, int64_t ws_bytes, int new_nnz, int new_users, int new_items, void* stream);

/* ---- rating sessions (csrc/session.cu, csrc/extract.cu, csrc/retrieve.cu) ----
 * A session scores one user from a rating row passed with the query, without changing the graph: session s is user
 * users[s] (>= G.num_users: a new user, starting from an empty row) with edits (s, item, value) applied to that user's
 * row only, in RatingGraph.update's encoding (value = label + 1 inserts or overwrites, 0 deletes, the last occurrence
 * of (s, item) wins; items must exist).  Only a pair's target user takes its row from the session; every other row and
 * column comes from G, so a session pair's subgraph, and its score, are bit-identical to those of the same pair on the
 * graph with the edits applied to that user. */
typedef struct {
  const int32_t* users;     /* [num_sessions] user id of each session (>= 0) */
  const int32_t* row_ptr;   /* [num_sessions+1] the merged rows */
  const int32_t* col_idx;   /* [row_ptr[num_sessions]] ascending within a row */
  const uint8_t* rating;    /* [row_ptr[num_sessions]] rating label */
  int32_t num_sessions;
  int32_t max_row_deg;      /* the longest session row */
} igmc_sessions_t;

/* Bytes of the workspace igmc_session_plan and igmc_session_apply share. */
int igmc_session_ws_bytes(int num_sessions, int D, int num_items, int64_t* bytes);

/* Validate (session in [0, num_sessions), item in [0, G->num_items), value 0..256, users >= 0, else IGMC_ERR_SESSIONS
 * in `err`), order the D edits by (session, item) keeping input order in a run, keep the last of each run, classify it
 * against the session's base row (binary search) and compute the rows' lengths and pointers into the workspace;
 * header [2] (device int64) = (total length, longest row).  Changes nothing in G. */
int igmc_session_plan(const igmc_csr_t* G, const int32_t* users, int num_sessions, const int32_t* sess,
                      const int32_t* items, const int32_t* values, int D, void* ws, int64_t ws_bytes, int64_t* header,
                      int* err, void* stream);

/* Merge every session row (a warp per session) into col_idx / rating [header[0]] and write row_ptr [num_sessions+1].
 * Same G, users, num_sessions, D and workspace as the plan, whose error word must be 0. */
int igmc_session_apply(const igmc_csr_t* G, const int32_t* users, int num_sessions, int D, void* ws, int64_t ws_bytes,
                       int32_t* row_ptr, int32_t* col_idx, uint8_t* rating, void* stream);

/* After igmc_candidate_pairs ran over the session rows as a CSR view (row_ptr / col_idx / rating of S, num_users =
 * num_sessions, num_items = G's, query users 0..num_sessions-1 or explicit pairs whose pair_u is the session index):
 * sess[i] = links_u[i] (the session), links_u[i] = users[sess[i]] and pair_id[i] = links_u[i] * num_items + links_v[i],
 * the pair id a graph with the edits applied samples the pair with.  tag is left as it is.  A session index out of
 * range sets IGMC_ERR_CANDIDATES. */
int igmc_session_pairs(const igmc_sessions_t* S, int num_items, int B, int32_t* links_u, const int32_t* links_v,
                       int64_t* pair_id, int32_t* sess, int* err, void* stream);

/* igmc_extract_batch in session mode: graph g takes its target user's row from session row sess[g] of S (the hop-1
 * item fringe, the visited marks of h > 1 and the target user's row scan) and everything else from G.  A session user
 * id >= G->num_users is never looked up in G's per-user structures.  `max_row_deg`: max(G's longest row, S's). */
int igmc_extract_sessions(const igmc_csr_t* G, const igmc_sessions_t* S, const int32_t* sess, const igmc_pairs_t* P,
                          int B, int h, int max_nodes_per_hop, double sample_ratio, uint64_t seed,
                          const uint64_t* seed_dev, int cap, const igmc_extract_ws_t* W, const float* class_values,
                          int num_classes, int max_row_deg, const igmc_batch_out_t* O, int* err, void* stream);

/* igmc_corated_items for sessions: query j is session j, its row N(u) the session row (pass 1 and the exclusion of
 * rated items), u' != u compared with the session's real user id; the columns come from G.  Workspace as
 * igmc_corated_ws_bytes(G->num_users, G->num_items, num_sessions, m). */
int igmc_corated_sessions(const igmc_csr_t* G, const igmc_sessions_t* S, int m, int exclude_rated, void* ws,
                          int64_t ws_bytes, int32_t* items, int32_t* paths, int* err, void* stream);

/* ---- online fine-tuning (csrc/online.cu; igmc_b200/train_eval.py: OnlineTrainer) ----
 * A trainer that follows graph updates draws each step's training pairs from G itself, a share of them from a ring of
 * recently rated pairs.  The ring holds `capacity` (user, item) pairs in ring_u / ring_v; `total` (device int64) counts
 * the pairs ever appended, so the window is its first W = min(total, capacity) slots.  Labels are never stored: a
 * window pair is looked up in G when it is drawn, so a later overwrite or delete is respected.
 *
 * igmc_online_recent_append appends the (users[i], items[i]) of every entry with values[i] > 0 of a delta (RatingGraph
 * update encoding) in input order at slot (total + rank) % capacity, the newest over the oldest, then total += their
 * count.  One CTA.  A negative id or a value outside 0..256 sets IGMC_ERR_GRAPH_UPDATE and the entry is skipped. */
int igmc_online_recent_append(const int32_t* users, const int32_t* items, const int32_t* values, int D, int32_t* ring_u,
                              int32_t* ring_v, int capacity, int64_t* total, int* err, void* stream);

/* One step's B training pairs for igmc_extract_batch (idx = NULL): links_u / links_v / label / pair_id [B] and seeds [3].
 * The step s = step_count[0] + step_ahead (step_count: the optimizer's device Adam step counter; step_ahead 1 when the
 * draw runs beside the step that will increment it, 0 otherwise), and
 *   seeds[0] = splitmix64(sample_seed + s)   the extraction sample seed, and the seed of the pair keys below
 *   seeds[1] = splitmix64(drop_seed + s)     the dropout seed of step s
 *   seeds[2] = splitmix64(drop_seed + s + 1) the dropout seed of step s + 1, the step that trains on these pairs
 * Slot j: key = sample_state(seeds[0], j, 0, 7) (csrc/common.cuh; hop slot 7 is never used by extraction).  When W > 0
 * and key >> 32 < recent_thresh (= round(recent_fraction * 2^32), 0..2^32) the pair is window entry
 * ((key & 0xffffffff) * W) >> 32, labelled by a binary search of its user's row; a window pair G does not hold (deleted,
 * or ids outside G) falls through.  Otherwise p = (h * nnz) >> 64 with h = sample_state(seeds[0], j, 1, 7) and nnz =
 * row_ptr[num_users]: user upper_bound(row_ptr[0..num_users], p) - 1, item col_idx[p], label rating[p].  pair_id = u *
 * num_items + v.  A graph without ratings sets IGMC_ERR_ONLINE (pairs (0, 0)).  Reads only device state: one captured
 * CUDA graph serves every step while G's shape stays. */
int igmc_online_draw(const igmc_csr_t* G, const int32_t* ring_u, const int32_t* ring_v, int capacity,
                     const int64_t* total, int64_t recent_thresh, const int64_t* step_count, int step_ahead,
                     uint64_t sample_seed, uint64_t drop_seed, int B, int32_t* links_u, int32_t* links_v, int32_t* label,
                     int64_t* pair_id, uint64_t* seeds, int* err, void* stream);

/* ---- Monte-Carlo-dropout draws (csrc/draws.cu; igmc_b200/recommend.py: predict_draws, recommend(draws=S)) ----
 * Draw s of pair (u, v) is a training-mode forward of the pair's enclosing subgraph with injected masks: each directed
 * edge kept with probability 1 - adj_dropout (the model's rate), each of the 128 hidden units before lin2 kept with
 * probability 0.5 and scaled by 2 (an injected hidden_keep stands for p = 0.5).  With pid = u * num_items + v, the
 * masks of draw s are counter hashes
 *   edges:  edge_keep(splitmix64(sample_state(draw_seed, pid, 0, 4) + s), e - edge_ptr[g], keep_thresh(adj_dropout))
 *   hidden: edge_keep(splitmix64(sample_state(draw_seed, pid, 1, 4) + s), o, keep_thresh(0.5))
 * (csrc/common.cuh, csrc/lists.cuh; hop slot 4 is used by neither extraction, hops 1..3, nor the online draw, hop 7).
 * edge_keep keeps iff the hash's high 32 bits reach the threshold, except that keep_thresh(1) = 0xFFFFFFFF keeps
 * nothing: at adj_dropout = 1 every edge is dropped, as the probability 1 - adj_dropout says.
 * A draw depends on (parameters, graph, pair, s, draw_seed) only, never on a batch position.  A batch of B graphs holds
 * G = B / S pairs times S consecutive draws, pair major; graphs G*S..B-1 are padding (tag -1).  The pair stream
 * (igmc_candidate_pairs) runs with G slots per batch.  1 <= S <= IGMC_DRAWS_MAX and S <= B. */
#define IGMC_DRAWS_MAX 256

/* Position i < G*S of the batch: pair g = i / S of the G pairs pair_u / pair_v / pair_pid / pair_tag, draw i - g*S;
 * positions G*S..B-1 copy pair 0 with tag -1 and draw 0.  Writes links_u / links_v / pair_id / tag / draw [B] for the
 * mapping kernels (igmc_item_query_pairs, igmc_session_pairs), which run next on all B positions, and for
 * igmc_extract_batch (idx = NULL). */
int igmc_draws_expand(int S, int B, const int32_t* pair_u, const int32_t* pair_v, const int64_t* pair_pid,
                      const int64_t* pair_tag, int32_t* links_u, int32_t* links_v, int64_t* pair_id, int64_t* tag,
                      int32_t* draw, void* stream);

/* For the batch O of B graphs extracted from those positions: edge_keep [O->edge_ptr[B]] and hidden_keep [B * 128] of
 * graph g from pair_id[g] and draw[g] by the hashes above; a graph with tag < 0 keeps everything.  One CTA per graph.
 * 0 <= adj_dropout <= 1 (else -2). */
int igmc_draws_mask(const igmc_batch_out_t* O, int B, const int64_t* pair_id, const int64_t* tag, const int32_t* draw,
                    float adj_dropout, uint64_t draw_seed, uint8_t* edge_keep, uint8_t* hidden_keep, void* stream);

/* Per pair g < G = B / S of the batch: its draws x_s = the fp32 checkpoint mean of preds[.][g*S + s] (as
 * igmc_topk_merge / igmc_score_scatter take it), then in fp64, in draw order and without fma contraction: mean = sum /
 * S, std = sqrt(sum (x_s - mean)^2 / (S - 1)) (0 when S = 1) and key = mean + beta * std, each rounded once to fp32.
 * A NaN draw makes all three NaN.  key != NULL: key [G] for every pair (igmc_topk_merge with K = 1 and B = G then
 * consumes it).  Otherwise, for t = tag[g*S] >= 0: value[t * S + s] = x_s, mean[t], std[t].  beta finite (else -2). */
int igmc_draws_stats(const float* preds, int K, int B, int S, const int64_t* tag, double beta, float* value,
                     float* mean, float* std, float* key, void* stream);

/* ---- counterfactual explanations (csrc/counterfactual.cu; igmc_b200/recommend.py: counterfactual) ----
 * Query q = (u, X, Y): which of u's own ratings, removed together, put item X behind the rival Y in recommend's order
 * (score descending, item ascending, NaN last)?  s_R(u, v) is the eval score of (u, v) on the graph with u's ratings at
 * the row positions R deleted: the pair extracted in session mode (igmc_extract_sessions) with u's row without R as the
 * target row, pair id u * num_items + v.  Greedy search from R = {}: pass 0 scores (u, X) and (u, Y) once; each later
 * pass scores every trial R + {i}, i a position of u's row not in R, and keeps the first trial by (X behind Y first,
 * then margin s(u,X) - s(u,Y) ascending with NaN after every number, then item ascending).  The search stops when X is
 * behind Y, when |R| = max_removals or when u's row has no position left.  A pass covers 2T positions, T = offsets[Q]
 * its trials (igmc_explain_offsets over count): position p is side p & 1 (0: X, 1: Y) of trial p >> 1. */
#define IGMC_COUNTERFACTUAL_MAX 256
typedef struct {
  const int32_t* users;     /* [num_query] u */
  const int32_t* items;     /* [num_query] X */
  const int32_t* rivals;    /* [num_query] Y */
  int32_t* size;            /* [num_query] |R| (0 before pass 1) */
  int32_t* removed;         /* [num_query, max_removals] R as positions in u's row, ascending */
  int32_t num_query, max_removals;
} igmc_counterfactual_t;

/* The pairs of positions [*cursor, *cursor + B), then *cursor += B (the igmc_candidate_pairs of a pass): position p
 * belongs to trial p >> 1 of query q (the last q with offsets[q] <= p >> 1), whose candidate (step > 0) is c = (p >> 1)
 * - offsets[q], the c-th position of u's row not in R.  Writes links_u = u, links_v = X or Y, pair_id = u * num_items +
 * links_v, tag = p (positions past 2T repeat the last one with tag -1), and per slot g its trial row as the session
 * rows igmc_extract_sessions reads with sess[g] = g: row_users[g] = u, row_ptr [B+1], and at [row_ptr[g],
 * row_ptr[g+1]) u's graph row without R and (step > 0) without the candidate, ascending, into row_col / row_rating
 * (row_cap entries; at most B * the longest graph row are needed).  Two launches.  Ids outside G, a candidate past the
 * row or rows beyond row_cap set IGMC_ERR_CANDIDATES. */
int igmc_counterfactual_pairs(const igmc_csr_t* G, const igmc_counterfactual_t* Q, const int64_t* offsets, int step,
                              int64_t* cursor, int B, int32_t* links_u, int32_t* links_v, int64_t* pair_id,
                              int64_t* tag, int32_t* row_users, int32_t* row_ptr, int32_t* row_col,
                              uint8_t* row_rating, int row_cap, int32_t* sess, int* err, void* stream);

/* One CTA per query q with trials in this pass (offsets[q+1] > offsets[q]), after the pass's scores are in
 * trial_scores [2T] (igmc_score_scatter by tag).  step 0: score / rival_score [q, 0] = the trial's two scores, found[q]
 * = X not ahead of Y.  step > 0: the query's first trial in the order above (a fixed-order block reduction) is
 * appended: its position joins removed, its item and label go to out_item / out_rating [q, size], its scores to
 * score / rival_score [q, size + 1], size += 1 and found[q] = X behind Y under it.  count[q] is the next pass's trial
 * count: deg(u) - size, or 0 once found, size = max_removals or the row has no position left; 0 for a query without
 * trials. */
int igmc_counterfactual_select(const igmc_csr_t* G, const igmc_counterfactual_t* Q, const int64_t* offsets,
                               const float* trial_scores, int step, int32_t* count, uint8_t* found, int32_t* out_item,
                               int32_t* out_rating, float* score, float* rival_score, int* err, void* stream);

/* ---- question impact for rating sessions (csrc/elicit.cu; igmc_b200/recommend.py: elicit, question_impact) ----
 * A question asks session s (igmc_sessions_t) about an item q not in s's row; its answers are the labels a = 0..A-1.
 * The trial row of (s, q, a) is s's row with (q, a) inserted at q's sorted position; x_a(t) is the eval score of
 * (users[s], t) extracted in session mode (igmc_extract_sessions) with that trial row as the target row, pair id
 * users[s] * num_items + t: bit for bit the score of a session with s's edits plus the edit (q, a + 1).  Targets
 * t_w, w < W: one list for every session (per_session = 0: targets [W]) or a row per session (per_session = 1:
 * targets [num_sessions, W]), -1 = an empty slot.  A unit (s, q) takes U = A * W consecutive batch positions, answer
 * major: position i of the unit is answer i / W and target slot i % W.  A batch of B positions holds G = B / U units
 * (U <= B); positions G*U..B-1 are padding, and so is the position of an empty target slot.  The unit stream
 * (igmc_candidate_pairs over the session rows as a CSR view, exclude_rated = 1, or over explicit (session, question)
 * pairs) runs with G slots per batch and writes unit_s (the session), unit_q (the question) and unit_tag. */

/* Position i < G*U, unit g = i / U, answer a = (i % U) / W, target t = the slot i % W of session unit_s[g]:
 * links_u = users[s], links_v = t, pair_id = links_u * num_items + links_v, tag = unit_tag[g] and sess = g * A + a
 * (the W targets of one answer share one trial row).  An empty slot, and every position G*U..B-1 (as unit 0, answer
 * 0), takes links_v = the unit's question and tag -1.  Trial row r = g * A + a, r < G * A: row_users[r] = users[s] and
 * at [row_ptr[r], row_ptr[r+1]) s's row with (q, a) inserted, ascending, into row_col / row_rating: the session rows
 * igmc_extract_sessions reads (row_ptr [G*A+1], row_cap entries; (B / W) * (the longest session row + 1) suffice).
 * Two launches: one CTA for the positions and the block scan of the row lengths deg(s) + 1, one CTA per trial row.
 * A session index, question or target outside its range (the unit then reads as session 0, question 0; the target
 * as an empty slot), a question already in the session's row, or rows past row_cap (cut short at row_cap) set
 * IGMC_ERR_CANDIDATES.  1 <= A <= 256, W >= 1, A * W <= B (else -1). */
int igmc_elicit_pairs(const igmc_sessions_t* S, int num_items, int A, const int32_t* targets, int W, int per_session,
                      const int32_t* unit_s, const int32_t* unit_q, const int64_t* unit_tag, int B, int32_t* links_u,
                      int32_t* links_v, int64_t* pair_id, int64_t* tag, int32_t* row_users, int32_t* row_ptr,
                      int32_t* row_col, uint8_t* row_rating, int row_cap, int32_t* sess, int* err, void* stream);

/* Per unit g < G of the batch, over its n real target slots w (tag[g*U + w] >= 0) in slot order: x_a(w) = the fp32
 * checkpoint mean of preds[.][g*U + a*W + w] (as igmc_topk_merge takes it), then in fp64 without fma contraction
 *   impact = sum_w (max_a x_a(w) - min_a x_a(w)) / n,   answer_mean[a] = sum_w x_a(w) / n,
 * each rounded once to fp32.  A NaN score of the unit makes its impact NaN, and the mean of its answer NaN.
 * key != NULL: key [G] = impact for every unit (igmc_topk_merge with K = 1 and B = G then consumes it; a unit without
 * real slots has key 0 and the merge skips its tag -1).  Otherwise, for the unit's tag t >= 0: impact[t] and
 * answer_mean[t * A + a]. */
int igmc_elicit_stats(const float* preds, int K, int B, int A, int W, const int64_t* tag, float* key, float* impact,
                      float* answer_mean, void* stream);

/* ---- cached top-k lists repaired after a rating-graph update (csrc/recommend_cache.cu; igmc_b200/recommend.py:
 * RecommendationCache) ----
 * With h = 1 the edits (a_i, b_i) of an update can change the enclosing subgraph, and so the score, only of the pairs
 * in ({a_i} x every item) U (every user x {b_i}) U (col(b_i) x row(a_i)) (DESIGN.md §19).  A cache keeps per query slot
 * j a list top_score / top_item [num_query, depth] whose leading entries (item >= 0) are an exact prefix of the slot's
 * ranking (igmc_topk_merge's order) and whose rest is padding (item -1, score -inf); complete[j] = 1 when the prefix
 * holds every candidate of the slot, else every unlisted candidate ranks after the last prefix entry. */

/* Workspace of igmc_rescore_plan: the candidate bitmap (ceil(num_items / 32) words), then per slot of a chunk one
 * bitmap row and two counts.  `bound` (<= 0: 256 MB) caps the bytes: past it the slots are processed in chunks of
 * *chunk (written when chunk != NULL); a workspace of any size runs in chunks of what it holds. */
int igmc_rescore_plan_ws_bytes(int num_query, int num_items, int64_t bound, int64_t* bytes, int* chunk);

/* The rescore plan of an update, on the UPDATED graph G: per query slot j (user users[j]) the sorted, distinct
 * candidate items of the affected set of the edits (edit_u[i], edit_v[i]) - every candidate when users[j] = some
 * edit_u[i]; else edit_v[i], and row(edit_u[i]) when users[j] rated edit_v[i] - in igmc_candidate_pairs' per_user
 * layout: user_off [num_query+1] int64 and out[user_off[j] ..) (out_cap entries; positions past it set
 * IGMC_ERR_CANDIDATES).  Candidates: `cand` [num_cand] ascending (NULL: every item), minus the user's rated items when
 * exclude_rated.  full[j] = 1 when every candidate of slot j is in its plan.  totals[0] = user_off[num_query],
 * totals[1] = the candidates of every slot (the pairs of a full ranking run).  A user bitmap row per slot built with
 * integer atomicOr, then a popcount scan: bit-identical across runs and chunk sizes.  Ids outside G set
 * IGMC_ERR_CANDIDATES (an edit is skipped, a slot has no candidates).  -2 when `ws_bytes` holds no slot. */
int igmc_rescore_plan(const igmc_csr_t* G, const int32_t* users, int num_query, const int32_t* edit_u,
                      const int32_t* edit_v, int num_edits, const int32_t* cand, int num_cand, int exclude_rated,
                      void* ws, int64_t ws_bytes, int64_t* user_off, int32_t* out, int64_t out_cap, uint8_t* full,
                      int64_t* totals, int* err, void* stream);

/* Before the merge of a repair, per slot j: the prefix without the items of out[user_off[j] .. user_off[j+1]) (binary
 * search; nothing is kept when full[j], since an edit of the slot's own user can change its candidates), compacted in order and padded to depth; the threshold key thr_score / thr_item [j] = the last prefix entry
 * before the removal, item -1 (none) when complete[j] or full[j], item -2 when the prefix is empty and the slot is
 * not complete (nothing is known to be exact).  1 <= depth <= IGMC_TOPK_MAX. */
int igmc_cache_invalidate(int num_query, int depth, const int64_t* user_off, const int32_t* resc, const uint8_t* full,
                          const uint8_t* complete, float* top_score, int64_t* top_item, float* thr_score,
                          int64_t* thr_item, void* stream);

/* After the merge (igmc_topk_merge of the rescored pairs into the invalidated lists), per slot j: its exact depth d -
 * every entry when the threshold is none, 0 for item -2, else the leading entries not ranked after the threshold key
 * (igmc_topk_merge's order) - with padding past d; complete[j] = (no threshold and d < depth); and the slots with a
 * threshold and d < k, ascending, in redo [*redo_count]: they are re-ranked over their whole catalogue.  One CTA.
 * 1 <= k <= depth <= IGMC_TOPK_MAX. */
int igmc_cache_settle(int num_query, int depth, int k, const float* thr_score, const int64_t* thr_item,
                      float* top_score, int64_t* top_item, uint8_t* complete, int32_t* redo, int32_t* redo_count,
                      void* stream);

/* Version / build info: returns the compiled SM arch (90) so the host can refuse stale builds. */
int igmc_build_info(void);

#ifdef __cplusplus
}
#endif
#endif
