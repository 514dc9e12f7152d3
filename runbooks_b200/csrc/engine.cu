// The fine-tune engine behind include/b200w.h: parameter / optimiser / activation memory for a
// Llama-family causal LM, the forward-loss-backward-clip-AdamW step as a sequence of the
// kernels in gemm.cu / attention.cu / ops.cu on one stream, and the data-parallel gradient
// all-reduce (NCCL, dlopen'ed) on a second stream overlapped with the last backward.
//
// Oracle for every stage: HF transformers 5.5.0 LlamaForCausalLM + the hand-written HF-Trainer
// step in oracle/ (SURVEY.md §8c): loss.backward(); clip_grad_norm_(1.0); AdamW.step().
#include <dlfcn.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/b200w.h"
#include "ctx_access.h"
#include "host_common.h"
#include "ops.h"
#include "ptx.cuh"

using namespace b200w;
using bf16 = __nv_bfloat16;

// ------------------------------------------------------------------------------------------
// NCCL through dlopen: the library must load (and export its symbols) on a box without NCCL.
// ------------------------------------------------------------------------------------------
namespace {
struct Uid { char internal[128]; };
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, /*ncclUniqueId by value*/ Uid, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*ReduceScatter)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*CommAbort)(void*) = nullptr;  // optional
  const char* (*GetErrorString)(int) = nullptr;
};
constexpr int kNcclInt64 = 4, kNcclFloat32 = 7, kNcclFloat64 = 8, kNcclBfloat16 = 9, kNcclSum = 0;

NcclApi& nccl() {
  static NcclApi api;
  if (!api.lib) {
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (api.lib) break;
    }
    if (!api.lib) throw Error(std::string("cannot dlopen libnccl: ") + dlerror());
    auto sym = [&](const char* s) {
      void* p = dlsym(api.lib, s);
      if (!p) throw Error(std::string("libnccl lacks symbol ") + s);
      return p;
    };
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(sym("ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(sym("ncclCommInitRank"));
    api.AllReduce = reinterpret_cast<decltype(api.AllReduce)>(sym("ncclAllReduce"));
    api.ReduceScatter = reinterpret_cast<decltype(api.ReduceScatter)>(sym("ncclReduceScatter"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(sym("ncclAllGather"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(sym("ncclCommDestroy"));
    api.CommAbort = reinterpret_cast<decltype(api.CommAbort)>(dlsym(api.lib, "ncclCommAbort"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(sym("ncclGetErrorString"));
  }
  return api;
}
#define B200W_NCCL(expr)                                                                  \
  do {                                                                                    \
    int _r = (expr);                                                                      \
    if (_r != 0) throw NcclError(std::string(#expr) + ": " + nccl().GetErrorString(_r));  \
  } while (0)
struct NcclError : Error { using Error::Error; };

std::string g_create_error;

struct Param {
  std::string name;
  int64_t rows, cols;    // shape of the HF tensor (what load_tensor / read_tensor exchange)
  int64_t irows, icols;  // shape on the device: equal, or with every head padded from dh to dhp
  size_t off;            // element offset into the flat parameter space
  bool is_norm;          // 1-D "ones" parameter (norm weight)
  bool is_zero_init;     // 1-D parameter HF initialises to zero (biases)
  bool decay;            // HF Trainer applies weight decay (trainer.py get_decay_parameter_names)
  int pad;               // 0 dense; 1 rows are heads of `dh` padded to `dhp`; 2 columns are
  size_t isize() const { return static_cast<size_t>(irows) * icols; }
};

// dst (internal, padded) <-> src (dense HF layout). Heads of dh elements sit at stride dhp along
// rows (pad == 1) or columns (pad == 2); the padding itself is never written here (it is zero from
// the memset at allocation and stays zero: every gradient that reaches it is exactly zero, see
// DESIGN.md 3.6).
__global__ void pad_scatter_kernel(const float* __restrict__ src, float* master, bf16* w, int64_t rows,
                                   int64_t cols, int64_t icols, int pad, int dh, int dhp) {
  const int64_t n = rows * cols;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / cols, c = i % cols;
    const int64_t ir = pad == 1 ? (r / dh) * dhp + r % dh : r;
    const int64_t ic = pad == 2 ? (c / dh) * dhp + c % dh : c;
    const float v = src[i];
    if (master) master[ir * icols + ic] = v;
    w[ir * icols + ic] = __float2bfloat16_rn(v);
  }
}
__global__ void pad_gather_kernel(const float* srcf, const bf16* srcb, float* __restrict__ dst,
                                  int64_t rows, int64_t cols, int64_t icols, int pad, int dh, int dhp) {
  const int64_t n = rows * cols;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / cols, c = i % cols;
    const int64_t ir = pad == 1 ? (r / dh) * dhp + r % dh : r;
    const int64_t ic = pad == 2 ? (c / dh) * dhp + c % dh : c;
    dst[i] = srcf ? srcf[ir * icols + ic] : __bfloat162float(srcb[ir * icols + ic]);
  }
}
// zero everything outside the real head dimensions of a padded parameter (after a random init)
__global__ void pad_zero_kernel(float* master, bf16* w, int64_t irows, int64_t icols, int pad, int dh,
                                int dhp) {
  const int64_t n = irows * icols;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / icols, c = i % icols;
    const bool is_pad = pad == 1 ? (r % dhp) >= dh : (c % dhp) >= dh;
    if (is_pad) {
      if (master) master[i] = 0.f;
      w[i] = __float2bfloat16_rn(0.f);
    }
  }
}
// inv_n[0] = 1 / count (0 when the count is 0): the loss normaliser, kept on the device
__global__ void set_count_kernel(long long* cnt, long long v) { cnt[0] = v; }
__global__ void inv_count_kernel(const long long* cnt, float* inv_n) {
  inv_n[0] = cnt[0] > 0 ? 1.f / static_cast<float>(cnt[0]) : 0.f;
}

// element j of the output holds the value of index i0 + j of the parameter's random stream (a rank that
// owns a slice of the fp32 master generates exactly the values the full tensor would hold there)
__global__ void init_normal_kernel(float* master, bf16* w, size_t n, uint64_t seed, float std, size_t i0 = 0) {
  for (size_t j = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; j < n;
       j += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t i = i0 + j;
    // splitmix64 counter hash -> two uniforms -> Box-Muller
    uint64_t z = seed + (i + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    const float u1 = (static_cast<uint32_t>(z >> 32) + 1.0f) * (1.0f / 4294967296.0f);
    const float u2 = static_cast<uint32_t>(z) * (1.0f / 4294967296.0f);
    const float r = sqrtf(-2.f * __logf(u1)) * __cosf(6.2831853f * u2) * std;
    if (master) master[j] = r;
    if (w) w[j] = __float2bfloat16_rn(r);
  }
}
// Fills this SM's shared memory (all 227 KB a block may use) with `pattern` (b200w_op_poison_onchip).
constexpr int POISON_SMEM = 227 * 1024;
__global__ void __launch_bounds__(128, 1) poison_onchip_kernel(uint32_t pattern) {
  extern __shared__ __align__(16) uint32_t poison_sm[];
  for (int i = threadIdx.x; i < POISON_SMEM / 4; i += blockDim.x) poison_sm[i] = pattern;
  __syncthreads();
  // keep the smem stores alive
  if (poison_sm[(threadIdx.x * 977) % (POISON_SMEM / 4)] != pattern) __trap();
}

__global__ void fill_kernel(float* master, bf16* w, size_t n, float val) {
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    if (master) master[i] = val;
    if (w) w[i] = __float2bfloat16_rn(val);
  }
}
}  // namespace

struct b200w_ctx {
  int device = 0;
  cudaStream_t stream = nullptr, comm_stream = nullptr;
  std::string err;
  int64_t launches = 0;
  int64_t dev_bytes = 0;
  std::vector<void*> allocs;

  // ---- model ----
  bool has_model = false, training = false;
  b200w_arch arch{};
  b200w_hparams hp{};
  int micro_batch = 0;
  int step = 0;
  int dhp = 128;   // head dimension on the device (head_dim 64 is stored zero-padded to 128)
  std::vector<Param> params;
  std::unordered_map<std::string, int> index;
  size_t n_elems = 0;       // all parameters
  size_t n_zero_prefix = 0; // embeddings + 1-D parameters: gradients accumulated, cleared per step
  struct Seg { size_t off, n; bool decay; };
  std::vector<Seg> segs;    // contiguous ranges of equal weight-decay policy, in offset order
  bf16* w = nullptr;
  float *master = nullptr, *m = nullptr, *v = nullptr, *g = nullptr;
  bf16* gw = nullptr;       // bf16 wire copy of the gradients (data parallel only)
  // Exchange ranges: the prefix's decay segments, then every matrix (the unit of the overlapped
  // gradient collective). With sharded optimiser state (training == 2) rank r owns slice r of every
  // range: master / m / v exist only for the owned slices, packed at offset range.off / nranks.
  struct Range { size_t off, cnt; bool decay; };
  std::vector<Range> ranges;
  bool shard = false;
  bool recompute = false;   // keep only every layer's input; the backward re-runs the layer's forward (B200W_TRAIN_RECOMPUTE)
  float2* rope_tab = nullptr;

  struct LayerP { size_t ln1, ln1b, ln2, ln2b, wqkv, bqkv, wo, bo, wgu, b1, wd, b2; };
  std::vector<LayerP> lp;
  size_t p_embed = 0, p_pos = 0, p_norm = 0, p_normb = 0, p_lm = 0;

  // ---- activations for one micro-batch ----
  struct LayerA {
    bf16 *h_in, *n1, *qkv, *attn, *h_mid, *n2, *gu, *act;
    float *rstd1, *rstd2, *mean1, *mean2, *lse;
  };
  std::vector<LayerA> la;
  bf16 *h_final = nullptr, *nf = nullptr, *logits = nullptr;
  float *rstdf = nullptr, *meanf = nullptr, *nll = nullptr;
  int32_t *ids_dev = nullptr, *labels_dev = nullptr, *targets = nullptr;
  size_t ids_cap = 0;
  int32_t* pinned = nullptr;
  size_t pinned_cap = 0;
  // per-document attention (the _docs calls): the batch's positions and the DocBounds derived from them
  int32_t *pos_dev = nullptr, *doc_start = nullptr, *doc_end = nullptr;
  size_t docs_cap = 0;
  bf16 *dh_a = nullptr, *dh_b = nullptr, *dn = nullptr, *dact = nullptr, *dgu = nullptr,
       *dattn = nullptr, *dqkv = nullptr;
  float *delta = nullptr, *dw_partial = nullptr;
  float* scal = nullptr;    // [0] loss, [1] gscale, [2] gnorm
  float* inv_n = nullptr;   // 1 / (global) target count of the running step
  long long* cnt_dev = nullptr;  // target count, summed over the ranks (HF num_items_in_batch)
  double* sumsq = nullptr;
  float* host_scal = nullptr;  // pinned [8]
  float* hook_scal = nullptr;

  // ---- timing / profiling (bench.py) ----
  cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;
  bool prof_gemm = false;
  std::vector<cudaEvent_t> prof_events;  // pairs
  size_t prof_used = 0;
  double prof_flops = 0;

  // ---- inference engine (infer.cu) ----
  void* infer = nullptr;
  void (*infer_destroy)(void*) = nullptr;

  // ---- DP ----
  void* comm = nullptr;
  int rank = 0, nranks = 1;
  int ar_sm_reserve = 0;  // SMs the GEMMs leave to NCCL while the all-reduce overlaps the backward
  bool poisoned = false;  // a CUDA / NCCL call failed: the context (and any collective) is dead
  cudaEvent_t ev_grad = nullptr, ev_comm = nullptr;

  template <typename T>
  T* alloc(size_t n) {
    void* p = nullptr;
    const size_t bytes = ((n * sizeof(T) + 255) / 256) * 256;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) {
      cudaGetLastError();
      throw std::bad_alloc();
    }
    allocs.push_back(p);
    dev_bytes += static_cast<int64_t>(bytes);
    return static_cast<T*>(p);
  }
  void release(void* p) {
    for (size_t i = 0; i < allocs.size(); ++i)
      if (allocs[i] == p) {
        cudaFree(p);
        allocs.erase(allocs.begin() + i);
        return;
      }
  }
  void free_all() {
    for (void* p : allocs) cudaFree(p);
    allocs.clear();
    dev_bytes = 0;
  }
};

namespace {

bool is_opt(const b200w_arch& a) { return a.family == B200W_FAMILY_OPT; }
bool is_falcon(const b200w_arch& a) { return a.family == B200W_FAMILY_FALCON; }
bool has_layernorm(const b200w_arch& a) { return is_opt(a) || is_falcon(a); }
// Llama's gate and up projections form one [2 f, d] matrix; OPT's fc1 and Falcon's dense_h_to_4h are [f, d]
bool gated_mlp(const b200w_arch& a) { return !is_opt(a) && !is_falcon(a); }
// the lm_head is the embedding matrix (OPT, Falcon)
bool tied_head(const b200w_ctx* c) { return c->p_lm == c->p_embed; }
int qd_of(const b200w_ctx* c) { return c->arch.num_heads * c->dhp; }
int kd_of(const b200w_ctx* c) { return c->arch.num_kv_heads * c->dhp; }
int qkv_dim(const b200w_ctx* c) { return qd_of(c) + 2 * kd_of(c); }
constexpr int OPT_POS_OFFSET = 2;  // HF models/opt/modeling_opt.py:53

// device scalar scratch for the per-kernel hooks (exists without a model)
float* ctx_scal(b200w_ctx* c) {
  if (!c->hook_scal) c->hook_scal = c->alloc<float>(8);
  return c->hook_scal;
}

template <typename F>
int guarded(b200w_ctx* ctx, F&& f) {
  if (!ctx) return B200W_ERR_INVALID;
  try {
    B200W_CUDA(cudaSetDevice(ctx->device));
    f();
    return B200W_OK;
  } catch (const NcclError& e) {
    ctx->err = e.what();
    ctx->poisoned = true;
    return B200W_ERR_NCCL;
  } catch (const std::bad_alloc&) {
    ctx->err = "device memory exhausted";
    return B200W_ERR_OOM;
  } catch (const Error& e) {
    ctx->err = e.what();
    if (ctx->err.rfind("check failed", 0) == 0) return B200W_ERR_INVALID;
    ctx->poisoned = true;
    return B200W_ERR_CUDA;
  } catch (const std::exception& e) {
    ctx->err = e.what();
    return B200W_ERR_INVALID;
  }
}

// kind: 'm' matrix (decayed), 'n' norm weight (ones, no decay), 'b' bias / LayerNorm bias (zeros, no
// decay). pad: see Param. HF Trainer's decay rule (trainer.py:1280-1290): everything except
// nn.LayerNorm parameters and names matching bias / layernorm / rmsnorm / norm.
void add_param(b200w_ctx* c, const std::string& name, int64_t rows, int64_t cols, char kind, size_t* off_out,
               int pad = 0) {
  const int dh = c->arch.head_dim, dhp = c->dhp;
  Param p{};
  p.name = name;
  p.rows = rows;
  p.cols = cols;
  p.irows = pad == 1 ? rows / dh * dhp : rows;
  p.icols = pad == 2 ? cols / dh * dhp : cols;
  p.off = c->n_elems;
  p.is_norm = kind == 'n';
  p.is_zero_init = kind == 'b';
  p.decay = kind == 'm';
  p.pad = dhp == dh ? 0 : pad;
  *off_out = c->n_elems;
  c->index[name] = static_cast<int>(c->params.size());
  c->params.push_back(p);
  c->n_elems += p.isize();
}

void build_segments(b200w_ctx* c) {
  c->segs.clear();
  for (const Param& p : c->params) {
    if (!c->segs.empty() && c->segs.back().decay == p.decay && c->segs.back().off + c->segs.back().n == p.off)
      c->segs.back().n += p.isize();
    else
      c->segs.push_back({p.off, p.isize(), p.decay});
  }
}

// ranges = the decay segments of the accumulated prefix + one range per fused matrix, in offset order
void build_ranges(b200w_ctx* c, const std::vector<std::pair<size_t, size_t>>& matrices) {
  c->ranges.clear();
  for (const auto& sg : c->segs) {
    if (sg.off >= c->n_zero_prefix) break;
    const size_t end = std::min(sg.off + sg.n, c->n_zero_prefix);
    c->ranges.push_back({sg.off, end - sg.off, sg.decay});
  }
  for (const auto& mtx : matrices) c->ranges.push_back({mtx.first, mtx.second, true});
}

void build_params_llama(b200w_ctx* c) {
  const b200w_arch& a = c->arch;
  const int d = a.hidden_size, f = a.intermediate_size, L = a.num_layers;
  const int qd = a.num_heads * a.head_dim, kd = a.num_kv_heads * a.head_dim;
  c->lp.assign(L, {});
  // atomically-accumulated gradients first, so one memset clears them
  add_param(c, "model.embed_tokens.weight", a.vocab_size, d, 'm', &c->p_embed);
  for (int l = 0; l < L; ++l) {
    const std::string pre = "model.layers." + std::to_string(l) + ".";
    add_param(c, pre + "input_layernorm.weight", 1, d, 'n', &c->lp[l].ln1);
    add_param(c, pre + "post_attention_layernorm.weight", 1, d, 'n', &c->lp[l].ln2);
  }
  add_param(c, "model.norm.weight", 1, d, 'n', &c->p_norm);
  c->n_zero_prefix = c->n_elems;
  size_t dummy;
  for (int l = 0; l < L; ++l) {
    const std::string pre = "model.layers." + std::to_string(l) + ".";
    // q, k, v rows are contiguous: together they are the fused [qkv_dim, d] projection
    add_param(c, pre + "self_attn.q_proj.weight", qd, d, 'm', &c->lp[l].wqkv);
    add_param(c, pre + "self_attn.k_proj.weight", kd, d, 'm', &dummy);
    add_param(c, pre + "self_attn.v_proj.weight", kd, d, 'm', &dummy);
    add_param(c, pre + "self_attn.o_proj.weight", d, qd, 'm', &c->lp[l].wo);
    // gate, up contiguous: the fused [2f, d] projection
    add_param(c, pre + "mlp.gate_proj.weight", f, d, 'm', &c->lp[l].wgu);
    add_param(c, pre + "mlp.up_proj.weight", f, d, 'm', &dummy);
    add_param(c, pre + "mlp.down_proj.weight", d, f, 'm', &c->lp[l].wd);
  }
  add_param(c, "lm_head.weight", a.vocab_size, d, 'm', &c->p_lm);
}

// OPT-125m layout (HF models/opt/modeling_opt.py; checkpoint keys of OPTForCausalLM). The tied
// lm_head is the embedding matrix itself (no separate parameter). q/k/v rows, their biases and the
// out_proj columns are stored with every 64-wide head padded to 128 (Param::pad).
void build_params_opt(b200w_ctx* c) {
  const b200w_arch& a = c->arch;
  const int d = a.hidden_size, f = a.intermediate_size, L = a.num_layers;
  const int qd = a.num_heads * a.head_dim;
  c->lp.assign(L, {});
  const std::string dec = "model.decoder.";
  add_param(c, dec + "embed_tokens.weight", a.vocab_size, d, 'm', &c->p_embed);
  add_param(c, dec + "embed_positions.weight", a.max_positions + OPT_POS_OFFSET, d, 'm', &c->p_pos);
  size_t dummy;
  for (int l = 0; l < L; ++l) {
    const std::string pre = dec + "layers." + std::to_string(l) + ".";
    auto& p = c->lp[l];
    add_param(c, pre + "self_attn_layer_norm.weight", 1, d, 'n', &p.ln1);
    add_param(c, pre + "self_attn_layer_norm.bias", 1, d, 'b', &p.ln1b);
    add_param(c, pre + "final_layer_norm.weight", 1, d, 'n', &p.ln2);
    add_param(c, pre + "final_layer_norm.bias", 1, d, 'b', &p.ln2b);
    add_param(c, pre + "self_attn.q_proj.bias", qd, 1, 'b', &p.bqkv, 1);
    add_param(c, pre + "self_attn.k_proj.bias", qd, 1, 'b', &dummy, 1);
    add_param(c, pre + "self_attn.v_proj.bias", qd, 1, 'b', &dummy, 1);
    add_param(c, pre + "self_attn.out_proj.bias", 1, d, 'b', &p.bo);
    add_param(c, pre + "fc1.bias", 1, f, 'b', &p.b1);
    add_param(c, pre + "fc2.bias", 1, d, 'b', &p.b2);
  }
  add_param(c, dec + "final_layer_norm.weight", 1, d, 'n', &c->p_norm);
  add_param(c, dec + "final_layer_norm.bias", 1, d, 'b', &c->p_normb);
  c->n_zero_prefix = c->n_elems;
  for (int l = 0; l < L; ++l) {
    const std::string pre = dec + "layers." + std::to_string(l) + ".";
    auto& p = c->lp[l];
    add_param(c, pre + "self_attn.q_proj.weight", qd, d, 'm', &p.wqkv, 1);
    add_param(c, pre + "self_attn.k_proj.weight", qd, d, 'm', &dummy, 1);
    add_param(c, pre + "self_attn.v_proj.weight", qd, d, 'm', &dummy, 1);
    add_param(c, pre + "self_attn.out_proj.weight", d, qd, 'm', &p.wo, 2);
    add_param(c, pre + "fc1.weight", f, d, 'm', &p.wgu);
    add_param(c, pre + "fc2.weight", d, f, 'm', &p.wd);
  }
  c->p_lm = c->p_embed;  // tied
}

// Falcon-7B layout (HF models/falcon/modeling_falcon.py, multi_query + parallel_attn, bias=False;
// checkpoint keys of FalconForCausalLM). query_key_value rows are [H q heads | 1 k head | 1 v head],
// every 64-wide head padded to 128 like OPT's; lm_head is tied to word_embeddings.
void build_params_falcon(b200w_ctx* c) {
  const b200w_arch& a = c->arch;
  const int d = a.hidden_size, f = a.intermediate_size, L = a.num_layers;
  const int qd = a.num_heads * a.head_dim, qkv = (a.num_heads + 2 * a.num_kv_heads) * a.head_dim;
  c->lp.assign(L, {});
  const std::string tr = "transformer.";
  add_param(c, tr + "word_embeddings.weight", a.vocab_size, d, 'm', &c->p_embed);
  for (int l = 0; l < L; ++l) {
    const std::string pre = tr + "h." + std::to_string(l) + ".";
    add_param(c, pre + "input_layernorm.weight", 1, d, 'n', &c->lp[l].ln1);
    add_param(c, pre + "input_layernorm.bias", 1, d, 'b', &c->lp[l].ln1b);
  }
  add_param(c, tr + "ln_f.weight", 1, d, 'n', &c->p_norm);
  add_param(c, tr + "ln_f.bias", 1, d, 'b', &c->p_normb);
  c->n_zero_prefix = c->n_elems;
  for (int l = 0; l < L; ++l) {
    const std::string pre = tr + "h." + std::to_string(l) + ".";
    auto& p = c->lp[l];
    add_param(c, pre + "self_attention.query_key_value.weight", qkv, d, 'm', &p.wqkv, 1);
    add_param(c, pre + "self_attention.dense.weight", d, qd, 'm', &p.wo, 2);
    add_param(c, pre + "mlp.dense_h_to_4h.weight", f, d, 'm', &p.wgu);
    add_param(c, pre + "mlp.dense_4h_to_h.weight", d, f, 'm', &p.wd);
  }
  c->p_lm = c->p_embed;  // tied
}

void alloc_activations(b200w_ctx* c) {
  const b200w_arch& a = c->arch;
  const bool opt = is_opt(a), falcon = is_falcon(a), ln = has_layernorm(a);
  const size_t T = static_cast<size_t>(c->micro_batch) * a.max_seq_len;
  const size_t d = a.hidden_size, f = a.intermediate_size, qd = qd_of(c), qkvd = qkv_dim(c),
               H = a.num_heads;
  const int L = a.num_layers;
  c->la.resize(L);
  // forward-only: every layer reuses one set. Recompute: one set too, but every layer keeps its own input
  const int Lsave = (c->training && !c->recompute) ? L : 1;
  for (int l = 0; l < L; ++l) {
    if (l < Lsave) {
      auto& x = c->la[l];
      x.h_in = c->alloc<bf16>(T * d);
      x.n1 = c->alloc<bf16>(T * d);
      x.qkv = c->alloc<bf16>(T * qkvd);
      x.attn = c->alloc<bf16>(T * qd);
      x.h_mid = c->alloc<bf16>(T * d);
      x.n2 = c->alloc<bf16>(T * d);
      x.gu = opt ? nullptr : c->alloc<bf16>(T * (falcon ? 1 : 2) * f);  // Falcon: the pre-GeLU activation
      x.act = c->alloc<bf16>(T * f);
      x.rstd1 = c->alloc<float>(T);
      x.rstd2 = c->alloc<float>(T);
      x.mean1 = ln ? c->alloc<float>(T) : nullptr;
      x.mean2 = opt ? c->alloc<float>(T) : nullptr;
      x.lse = c->alloc<float>(H * T);
    } else {
      c->la[l] = c->la[0];
      if (c->training && c->recompute) c->la[l].h_in = c->alloc<bf16>(T * d);
    }
  }
  c->h_final = c->alloc<bf16>(T * d);
  c->nf = c->alloc<bf16>(T * d);
  c->rstdf = c->alloc<float>(T);
  if (ln) c->meanf = c->alloc<float>(T);
  c->logits = c->alloc<bf16>(T * a.vocab_size);
  c->nll = c->alloc<float>(T);
  c->targets = c->alloc<int32_t>(T);
  c->scal = c->alloc<float>(8);
  c->inv_n = c->alloc<float>(1);
  c->cnt_dev = c->alloc<long long>(1);
  c->sumsq = c->alloc<double>(1);
  if (c->training) {
    c->dh_a = c->alloc<bf16>(T * d);
    c->dh_b = c->alloc<bf16>(T * d);
    c->dn = c->alloc<bf16>(T * d);
    c->dact = c->alloc<bf16>(T * f);
    if (!ln) c->dgu = c->alloc<bf16>(T * 2 * f);
    c->dattn = c->alloc<bf16>(T * qd);
    c->dqkv = c->alloc<bf16>(T * qkvd);
    c->delta = c->alloc<float>(H * T);
    // norm backward partials [blocks, d] (RMSNorm) or [blocks, 2 d] (LayerNorm); bias column sums
    // [colsum_blocks, widest projection]
    size_t part = static_cast<size_t>(rmsnorm_bwd_blocks(static_cast<int>(T))) * d * (ln ? 2 : 1);
    if (opt) {
      const size_t widest = std::max<size_t>({qkvd, f, d});
      part = std::max(part, static_cast<size_t>(colsum_blocks(static_cast<int>(T))) * widest);
    }
    c->dw_partial = c->alloc<float>(part);
  }
  if (!opt) {  // the table is over the real head_dim; padded heads rotate their first head_dim columns
    c->rope_tab = c->alloc<float2>(static_cast<size_t>(a.max_seq_len) * (a.head_dim / 2));
    rope_table(c->rope_tab, a.max_seq_len, a.head_dim, a.rope_theta, c->stream);
  }
}

// GEMM launch with optional CUDA-event bracketing (bench.py's roofline leg)
void egemm(b200w_ctx* c, const void* A, bool a_mn, int lda, const void* B, bool b_mn, int ldb, void* D,
           const void* C, bool out_fp32, int ldd, int M, int N, int K, const void* bias = nullptr, int act = 0,
           void* d2_bf16 = nullptr) {
  cudaStream_t s = c->stream;
  if (c->prof_gemm) {
    if (c->prof_used + 2 > c->prof_events.size()) {
      for (int i = 0; i < 2; ++i) {
        cudaEvent_t e;
        B200W_CUDA(cudaEventCreate(&e));
        c->prof_events.push_back(e);
      }
    }
    B200W_CUDA(cudaEventRecord(c->prof_events[c->prof_used], s));
  }
  gemm_bf16_ex(A, a_mn, lda, B, b_mn, ldb, D, C, out_fp32, ldd, M, N, K, 0, bias, act, s, d2_bf16);
  ++c->launches;
  if (c->prof_gemm) {
    B200W_CUDA(cudaEventRecord(c->prof_events[c->prof_used + 1], s));
    c->prof_used += 2;
    c->prof_flops += 2.0 * M * N * static_cast<double>(K);
  }
}

// ---- forward of one micro-batch (ids already on device) ------------------------------------------
// The shapes of a micro-batch of nseq sequences. qd / kd / qkvd are over the device's head width dhp; dh is the
// model's head_dim, which sets the attention scale and the RoPE width.
struct Dims {
  int nseq, S, T, d, f, H, Hkv, dh, qd, kd, qkvd, V;
  float scale, eps;
  Dims(const b200w_ctx* c, int n_seqs)
      : nseq(n_seqs), S(c->arch.max_seq_len), T(nseq * S), d(c->arch.hidden_size), f(c->arch.intermediate_size),
        H(c->arch.num_heads), Hkv(c->arch.num_kv_heads), dh(c->arch.head_dim), qd(qd_of(c)), kd(kd_of(c)),
        qkvd(qkv_dim(c)), V(c->arch.vocab_size), scale(1.f / sqrtf(static_cast<float>(dh))),
        eps(c->arch.rms_norm_eps) {}
};

// One Llama decoder layer: c->la[l] receives the activations the backward needs, h_next the layer's output
// (nullptr in the recompute pass of the backward, which stops before the down projection).
// docs (nullable): RoPE at the documents' positions and attention within each document.
void forward_layer_llama(b200w_ctx* c, const Dims& m, int l, const bf16* h_in, bf16* h_next, const DocBounds* docs) {
  cudaStream_t s = c->stream;
  int64_t& n = c->launches;
  auto& x = c->la[l];
  const auto& p = c->lp[l];
  rmsnorm_fwd(h_in, c->w + p.ln1, x.n1, x.rstd1, m.T, m.d, m.eps, s); ++n;
  egemm(c, x.n1, false, m.d, c->w + p.wqkv, false, m.d, x.qkv, nullptr, false, m.qkvd, m.T, m.qkvd, m.d);
  rope_apply(x.qkv, m.qkvd, c->rope_tab, m.T, m.S, m.H + m.Hkv, m.dh, false, s, 0, docs ? docs->pos : nullptr); ++n;
  attention_fwd(x.qkv, m.qkvd, m.qd, m.qd + m.kd, x.attn, m.qd, x.lse, m.nseq, m.S, m.H, m.Hkv, m.scale, s, docs); ++n;
  egemm(c, x.attn, false, m.qd, c->w + p.wo, false, m.qd, x.h_mid, h_in, false, m.d, m.T, m.d, m.qd);
  rmsnorm_fwd(x.h_mid, c->w + p.ln2, x.n2, x.rstd2, m.T, m.d, m.eps, s); ++n;
  egemm(c, x.n2, false, m.d, c->w + p.wgu, false, m.d, x.gu, nullptr, false, 2 * m.f, m.T, 2 * m.f, m.d);
  swiglu_fwd(x.gu, x.act, m.T, m.f, s); ++n;
  if (h_next) egemm(c, x.act, false, m.f, c->w + p.wd, false, m.f, h_next, x.h_mid, false, m.d, m.T, m.d, m.f);
}

// OPT decoder layer (HF models/opt/modeling_opt.py OPTDecoderLayer, pre-LN).
// q is scaled by head_dim^-0.5 inside the attention kernel (HF scales q after q_proj and calls the
// attention with scaling 1.0: the same product, and the factor 1/8 is exact in bf16).
void forward_layer_opt(b200w_ctx* c, const Dims& m, int l, const bf16* h_in, bf16* h_next) {
  cudaStream_t s = c->stream;
  int64_t& n = c->launches;
  auto& x = c->la[l];
  const auto& p = c->lp[l];
  layernorm_fwd(h_in, c->w + p.ln1, c->w + p.ln1b, x.n1, x.mean1, x.rstd1, m.T, m.d, m.eps, s); ++n;
  // nn.Linear(bias=True): the bias (and fc1's ReLU) ride in the GEMM epilogue, added in fp32 before the one
  // rounding to bf16
  egemm(c, x.n1, false, m.d, c->w + p.wqkv, false, m.d, x.qkv, nullptr, false, m.qkvd, m.T, m.qkvd, m.d,
        c->w + p.bqkv, 0);
  attention_fwd(x.qkv, m.qkvd, m.qd, m.qd + m.kd, x.attn, m.qd, x.lse, m.nseq, m.S, m.H, m.Hkv, m.scale, s); ++n;
  egemm(c, x.attn, false, m.qd, c->w + p.wo, false, m.qd, x.h_mid, h_in, false, m.d, m.T, m.d, m.qd, c->w + p.bo, 0);
  layernorm_fwd(x.h_mid, c->w + p.ln2, c->w + p.ln2b, x.n2, x.mean2, x.rstd2, m.T, m.d, m.eps, s); ++n;
  egemm(c, x.n2, false, m.d, c->w + p.wgu, false, m.d, x.act, nullptr, false, m.f, m.T, m.f, m.d, c->w + p.b1, 1);  // ReLU
  egemm(c, x.act, false, m.f, c->w + p.wd, false, m.f, h_next, x.h_mid, false, m.d, m.T, m.d, m.f, c->w + p.b2, 0);
}

// Falcon decoder layer (HF models/falcon/modeling_falcon.py FalconDecoderLayer.forward :580-650 with
// parallel_attn and one input_layernorm): ln = LN(h); h' = h + dense(attn(ln)) + 4h_to_h(gelu(h_to_4h(ln))).
// Multi-query attention: H query heads share one key/value head (the GQA path with Hkv = 1).
void forward_layer_falcon(b200w_ctx* c, const Dims& m, int l, const bf16* h_in, bf16* h_next) {
  cudaStream_t s = c->stream;
  int64_t& n = c->launches;
  auto& x = c->la[l];
  const auto& p = c->lp[l];
  layernorm_fwd(h_in, c->w + p.ln1, c->w + p.ln1b, x.n1, x.mean1, x.rstd1, m.T, m.d, m.eps, s); ++n;
  egemm(c, x.n1, false, m.d, c->w + p.wqkv, false, m.d, x.qkv, nullptr, false, m.qkvd, m.T, m.qkvd, m.d);
  rope_apply(x.qkv, m.qkvd, c->rope_tab, m.T, m.S, m.H + m.Hkv, m.dh, false, s, c->dhp); ++n;
  attention_fwd(x.qkv, m.qkvd, m.qd, m.qd + m.kd, x.attn, m.qd, x.lse, m.nseq, m.S, m.H, m.Hkv, m.scale, s); ++n;
  egemm(c, x.attn, false, m.qd, c->w + p.wo, false, m.qd, x.h_mid, h_in, false, m.d, m.T, m.d, m.qd);
  egemm(c, x.n1, false, m.d, c->w + p.wgu, false, m.d, x.gu, nullptr, false, m.f, m.T, m.f, m.d);
  gelu_fwd(x.gu, x.act, static_cast<size_t>(m.T) * m.f, s); ++n;
  egemm(c, x.act, false, m.f, c->w + p.wd, false, m.f, h_next, x.h_mid, false, m.d, m.T, m.d, m.f);
}

// docs: Llama family only (check_docs_family refuses the others before any GPU work)
void forward_micro(b200w_ctx* c, const int32_t* ids, int nseq, const DocBounds* docs = nullptr) {
  const Dims m(c, nseq);
  const bool opt = is_opt(c->arch), falcon = is_falcon(c->arch);
  cudaStream_t s = c->stream;
  int64_t& n = c->launches;
  const int L = c->arch.num_layers;

  bf16* h = c->la[0].h_in;
  embed_fwd(ids, c->w + c->p_embed, opt ? c->w + c->p_pos : nullptr, h, m.T, m.d, m.V, m.S,
            opt ? OPT_POS_OFFSET : 0, s); ++n;
  for (int l = 0; l < L; ++l) {
    bf16* h_in = c->training ? c->la[l].h_in : h;
    bf16* h_next = c->training ? (l + 1 < L ? c->la[l + 1].h_in : c->h_final)
                               : (h == c->la[0].h_in ? c->h_final : c->la[0].h_in);
    if (opt) forward_layer_opt(c, m, l, h_in, h_next);
    else if (falcon) forward_layer_falcon(c, m, l, h_in, h_next);
    else forward_layer_llama(c, m, l, h_in, h_next, docs);
    h = h_next;
  }
  // in training mode h == h_final; in forward-only mode h is whichever buffer came last
  if (has_layernorm(c->arch))
    layernorm_fwd(h, c->w + c->p_norm, c->w + c->p_normb, c->nf, c->meanf, c->rstdf, m.T, m.d, m.eps, s);
  else
    rmsnorm_fwd(h, c->w + c->p_norm, c->nf, c->rstdf, m.T, m.d, m.eps, s);
  ++n;
  egemm(c, c->nf, false, m.d, c->w + c->p_lm, false, m.d, c->logits, nullptr, false, m.V, m.T, m.V, m.d);
  if (c->training && h != c->h_final) throw Error("internal: residual stream bookkeeping");
}

// loss + dlogits (in place); the normaliser 1 / num_items_in_batch is the device scalar c->inv_n
void loss_micro(b200w_ctx* c, const int32_t* labels, int nseq) {
  const Dims m(c, nseq);
  cudaStream_t s = c->stream;
  ce_shift_targets(labels, c->targets, m.T, m.S, s); ++c->launches;
  ce_loss_fwd_bwd(c->logits, c->targets, c->nll, m.T, m.V, c->inv_n, s); ++c->launches;
  reduce_sum_f32(c->nll, c->scal + 0, m.T, c->inv_n, s); ++c->launches;
}

// B200W_AR_MODE (debugging aid, same arithmetic in every mode):
//   overlap (default)  per-matrix all-reduce on comm_stream as soon as the last micro-step's backward
//                      has produced the gradient, concurrent with the rest of the backward
//   sync               as overlap, but the host drains c->stream before enqueuing each all-reduce
//   serial             per-matrix, but c->stream waits for each all-reduce: never concurrent with compute
//   end                one all-reduce of the whole gradient after the backward
// Overlap is the default for every rank count.
enum class ArMode { Overlap, Sync, Serial, End };
ArMode ar_mode() {
  const char* m = getenv("B200W_AR_MODE");
  const std::string v = m ? m : "";
  if (v == "end") return ArMode::End;
  if (v == "sync") return ArMode::Sync;
  if (v == "serial") return ArMode::Serial;
  return ArMode::Overlap;
}

void ensure_wire(b200w_ctx* c) {
  if (!c->gw) c->gw = c->alloc<bf16>(c->n_elems);
}

// Gradient exchange of the flat range [off, off + count): the fp32 accumulation buffer is rounded to
// bf16 into the wire copy (main stream), and the wire copy is summed over the ranks by NCCL on the
// comm stream (13.5 GB per step for Llama-2-7B instead of 27 GB; SURVEY.md 8 a11). The optimiser
// then reads the reduced bf16 gradients directly.
// Sharded optimiser state: the collective is a reduce-scatter -- rank r receives the sum of slice r of
// the range, in place, which is all its share of the optimiser needs (SURVEY.md 8e, config #5:
// reduce_scatter -> local AdamW on the shard -> all_gather, the wire bytes of one all-reduce).
// precast: the wgrad GEMM that produced this range already wrote its bf16 wire copy (EpiExtra::d2).
void exchange_one(b200w_ctx* c, size_t off, size_t count, bool precast = false) {
  const ArMode mode = ar_mode();
  if (!precast) { cast_f32_to_bf16(c->g + off, c->gw + off, count, c->stream); ++c->launches; }
  if (mode == ArMode::Sync) B200W_CUDA(cudaStreamSynchronize(c->stream));
  B200W_CUDA(cudaEventRecord(c->ev_grad, c->stream));
  B200W_CUDA(cudaStreamWaitEvent(c->comm_stream, c->ev_grad, 0));
  if (c->shard) {
    const size_t n = count / c->nranks;
    B200W_NCCL(nccl().ReduceScatter(c->gw + off, c->gw + off + c->rank * n, n, kNcclBfloat16, kNcclSum, c->comm,
                                    c->comm_stream));
  } else {
    B200W_NCCL(nccl().AllReduce(c->gw + off, c->gw + off, count, kNcclBfloat16, kNcclSum, c->comm,
                                c->comm_stream));
  }
  ++c->launches;
  if (mode == ArMode::Serial) {
    B200W_CUDA(cudaEventRecord(c->ev_comm, c->comm_stream));
    B200W_CUDA(cudaStreamWaitEvent(c->stream, c->ev_comm, 0));
  }
}
void allreduce_range(b200w_ctx* c, size_t off, size_t count, bool precast = false) {
  if (count == 0) return;
  if (!c->shard) return exchange_one(c, off, count, precast);
  // sharded: slices are defined per exchange range, so a request is served range by range
  bool any = false;
  for (const auto& r : c->ranges)
    if (r.off >= off && r.off + r.cnt <= off + count) { exchange_one(c, r.off, r.cnt, precast); any = true; }
  if (!any) throw Error("internal: gradient exchange request does not match the exchange ranges");
}

// Where one micro-step's weight gradients go. first: the micro-step overwrites the gradients instead of
// accumulating them. overlap_ar: each range's gradient exchange starts as soon as the range is final.
struct GradOut {
  b200w_ctx* c;
  int T;
  bool first, overlap_ar;
  // dW [M, N] (+)= dy[T, M]^T x[T, N] into the gradient at off, then the exchange of that matrix; the GEMM epilogue
  // writes its bf16 wire copy itself
  void wgrad(size_t off, const void* dy, int M, const void* x, int N) const {
    egemm(c, dy, true, M, x, true, N, c->g + off, first ? nullptr : c->g + off, true, N, M, N, T, nullptr, 0,
          overlap_ar ? c->gw + off : nullptr);
    if (overlap_ar) allreduce_range(c, off, static_cast<size_t>(M) * N, true);
  }
  void exchange(size_t off, size_t count) const {
    if (overlap_ar) allreduce_range(c, off, count);
  }
};

// The backward of one decoder layer takes the gradient of its output in dh_cur and leaves the gradient of its
// input there; dh_alt is the other buffer of the pair.
void backward_layer_llama(b200w_ctx* c, const Dims& m, const GradOut& go, int l, bf16*& dh_cur, bf16*& dh_alt,
                          const DocBounds* docs) {
  cudaStream_t s = c->stream;
  int64_t& n = c->launches;
  float* g = c->g;
  auto& x = c->la[l];
  const auto& p = c->lp[l];
  // activation recomputation: the layer's forward again, from its saved input into the shared buffers (the same
  // kernels on the same operands: bit-identical activations, hence bit-identical gradients)
  if (c->recompute) forward_layer_llama(c, m, l, x.h_in, nullptr, docs);
  // h_next = h_mid + act Wd^T
  egemm(c, dh_cur, false, m.d, c->w + p.wd, true, m.f, c->dact, nullptr, false, m.f, m.T, m.f, m.d);
  go.wgrad(p.wd, dh_cur, m.d, x.act, m.f);
  swiglu_bwd(c->dact, x.gu, c->dgu, m.T, m.f, s); ++n;
  egemm(c, c->dgu, false, 2 * m.f, c->w + p.wgu, true, m.d, c->dn, nullptr, false, m.d, m.T, m.d, 2 * m.f);
  go.wgrad(p.wgu, c->dgu, 2 * m.f, x.n2, m.d);
  // dh_mid = dh + rmsnorm_bwd(dn2)
  rmsnorm_bwd(c->dn, x.h_mid, c->w + p.ln2, x.rstd2, dh_cur, dh_alt, g + p.ln2, c->dw_partial, m.T, m.d, s); n += 2;
  std::swap(dh_cur, dh_alt);
  // h_mid = h_in + attn Wo^T
  egemm(c, dh_cur, false, m.d, c->w + p.wo, true, m.qd, c->dattn, nullptr, false, m.qd, m.T, m.qd, m.d);
  go.wgrad(p.wo, dh_cur, m.d, x.attn, m.qd);
  attention_bwd(x.qkv, m.qkvd, m.qd, m.qd + m.kd, x.attn, c->dattn, m.qd, x.lse, c->delta, c->dqkv, m.nseq, m.S,
                m.H, m.Hkv, m.scale, s, docs); n += 3;
  rope_apply(c->dqkv, m.qkvd, c->rope_tab, m.T, m.S, m.H + m.Hkv, m.dh, true, s, 0, docs ? docs->pos : nullptr); ++n;
  egemm(c, c->dqkv, false, m.qkvd, c->w + p.wqkv, true, m.d, c->dn, nullptr, false, m.d, m.T, m.d, m.qkvd);
  go.wgrad(p.wqkv, c->dqkv, m.qkvd, x.n1, m.d);
  rmsnorm_bwd(c->dn, x.h_in, c->w + p.ln1, x.rstd1, dh_cur, dh_alt, g + p.ln1, c->dw_partial, m.T, m.d, s); n += 2;
  std::swap(dh_cur, dh_alt);
}

// OPT: bias gradients are column sums of the projection's output gradient.
void backward_layer_opt(b200w_ctx* c, const Dims& m, const GradOut& go, int l, bf16*& dh_cur, bf16*& dh_alt) {
  cudaStream_t s = c->stream;
  int64_t& n = c->launches;
  float* g = c->g;
  float* part = c->dw_partial;
  auto& x = c->la[l];
  const auto& p = c->lp[l];
  // h_next = h_mid + act W2^T + b2
  colsum_add(dh_cur, g + p.b2, part, m.T, m.d, m.d, s); n += 2;
  egemm(c, dh_cur, false, m.d, c->w + p.wd, true, m.f, c->dact, nullptr, false, m.f, m.T, m.f, m.d);
  go.wgrad(p.wd, dh_cur, m.d, x.act, m.f);
  // act = relu(n2 W1^T + b1)
  relu_bwd(c->dact, x.act, c->dact, static_cast<size_t>(m.T) * m.f, s); ++n;
  colsum_add(c->dact, g + p.b1, part, m.T, m.f, m.f, s); n += 2;
  egemm(c, c->dact, false, m.f, c->w + p.wgu, true, m.d, c->dn, nullptr, false, m.d, m.T, m.d, m.f);
  go.wgrad(p.wgu, c->dact, m.f, x.n2, m.d);
  layernorm_bwd(c->dn, x.h_mid, c->w + p.ln2, x.mean2, x.rstd2, dh_cur, dh_alt, g + p.ln2, g + p.ln2b, part,
                m.T, m.d, s); n += 3;
  std::swap(dh_cur, dh_alt);
  // h_mid = h_in + attn Wo^T + bo
  colsum_add(dh_cur, g + p.bo, part, m.T, m.d, m.d, s); n += 2;
  egemm(c, dh_cur, false, m.d, c->w + p.wo, true, m.qd, c->dattn, nullptr, false, m.qd, m.T, m.qd, m.d);
  go.wgrad(p.wo, dh_cur, m.d, x.attn, m.qd);
  attention_bwd(x.qkv, m.qkvd, m.qd, m.qd + m.kd, x.attn, c->dattn, m.qd, x.lse, c->delta, c->dqkv, m.nseq, m.S,
                m.H, m.Hkv, m.scale, s); n += 3;
  colsum_add(c->dqkv, g + p.bqkv, part, m.T, m.qkvd, m.qkvd, s); n += 2;
  egemm(c, c->dqkv, false, m.qkvd, c->w + p.wqkv, true, m.d, c->dn, nullptr, false, m.d, m.T, m.d, m.qkvd);
  go.wgrad(p.wqkv, c->dqkv, m.qkvd, x.n1, m.d);
  layernorm_bwd(c->dn, x.h_in, c->w + p.ln1, x.mean1, x.rstd1, dh_cur, dh_alt, g + p.ln1, g + p.ln1b, part,
                m.T, m.d, s); n += 3;
  std::swap(dh_cur, dh_alt);
}

// Falcon: both branches read the same LayerNorm output, so its gradient is the sum of the MLP branch's (written
// first) and the attention branch's (accumulated by the qkv dgrad GEMM's C operand).
void backward_layer_falcon(b200w_ctx* c, const Dims& m, const GradOut& go, int l, bf16*& dh_cur, bf16*& dh_alt) {
  cudaStream_t s = c->stream;
  int64_t& n = c->launches;
  float* g = c->g;
  auto& x = c->la[l];
  const auto& p = c->lp[l];
  // MLP branch: h' += gelu(ln W1^T) W2^T
  egemm(c, dh_cur, false, m.d, c->w + p.wd, true, m.f, c->dact, nullptr, false, m.f, m.T, m.f, m.d);
  go.wgrad(p.wd, dh_cur, m.d, x.act, m.f);
  gelu_bwd(c->dact, x.gu, c->dact, static_cast<size_t>(m.T) * m.f, s); ++n;
  egemm(c, c->dact, false, m.f, c->w + p.wgu, true, m.d, c->dn, nullptr, false, m.d, m.T, m.d, m.f);
  go.wgrad(p.wgu, c->dact, m.f, x.n1, m.d);
  // attention branch: h' += attn Wo^T
  egemm(c, dh_cur, false, m.d, c->w + p.wo, true, m.qd, c->dattn, nullptr, false, m.qd, m.T, m.qd, m.d);
  go.wgrad(p.wo, dh_cur, m.d, x.attn, m.qd);
  attention_bwd(x.qkv, m.qkvd, m.qd, m.qd + m.kd, x.attn, c->dattn, m.qd, x.lse, c->delta, c->dqkv, m.nseq, m.S,
                m.H, m.Hkv, m.scale, s); n += 3;
  rope_apply(c->dqkv, m.qkvd, c->rope_tab, m.T, m.S, m.H + m.Hkv, m.dh, true, s, c->dhp); ++n;
  egemm(c, c->dqkv, false, m.qkvd, c->w + p.wqkv, true, m.d, c->dn, c->dn, false, m.d, m.T, m.d, m.qkvd);
  go.wgrad(p.wqkv, c->dqkv, m.qkvd, x.n1, m.d);
  layernorm_bwd(c->dn, x.h_in, c->w + p.ln1, x.mean1, x.rstd1, dh_cur, dh_alt, g + p.ln1, g + p.ln1b,
                c->dw_partial, m.T, m.d, s); n += 3;
  std::swap(dh_cur, dh_alt);
}

// backward of one micro-batch. first: overwrite gradients instead of accumulating.
// overlap_ar: launch the all-reduce of each matrix as soon as its gradient is final.
void backward_micro(b200w_ctx* c, const int32_t* ids, int nseq, bool first, bool overlap_ar,
                    const DocBounds* docs) {
  const Dims m(c, nseq);
  const b200w_arch& a = c->arch;
  const bool opt = is_opt(a), falcon = is_falcon(a);
  cudaStream_t s = c->stream;
  int64_t& n = c->launches;
  float* g = c->g;
  const GradOut go{c, m.T, first, overlap_ar};
  // while the all-reduce runs under the backward, the persistent GEMMs leave NCCL its SMs
  if (overlap_ar) gemm_set_sm_reserve(c->ar_sm_reserve);
  try {
    // lm_head: dnf = dlogits W ; dW += dlogits^T nf
    egemm(c, c->logits, false, m.V, c->w + c->p_lm, true, m.d, c->dn, nullptr, false, m.d, m.T, m.d, m.V);
    // A tied head's gradient is the embedding's, zeroed with the prefix at the start of the step: the wgrad always
    // accumulates, embed_bwd adds the lookup rows to it, and it is exchanged with the prefix.
    if (tied_head(c))
      egemm(c, c->logits, true, m.V, c->nf, true, m.d, g + c->p_lm, g + c->p_lm, true, m.d, m.V, m.d, m.T);
    else
      go.wgrad(c->p_lm, c->logits, m.V, c->nf, m.d);
    bf16* dh_cur = c->dh_a;
    bf16* dh_alt = c->dh_b;
    if (has_layernorm(a)) {
      layernorm_bwd(c->dn, c->h_final, c->w + c->p_norm, c->meanf, c->rstdf, nullptr, dh_cur, g + c->p_norm,
                    g + c->p_normb, c->dw_partial, m.T, m.d, s); n += 3;
    } else {
      rmsnorm_bwd(c->dn, c->h_final, c->w + c->p_norm, c->rstdf, nullptr, dh_cur, g + c->p_norm, c->dw_partial,
                  m.T, m.d, s); n += 2;
    }
    for (int l = a.num_layers - 1; l >= 0; --l) {
      if (opt) backward_layer_opt(c, m, go, l, dh_cur, dh_alt);
      else if (falcon) backward_layer_falcon(c, m, go, l, dh_cur, dh_alt);
      else backward_layer_llama(c, m, go, l, dh_cur, dh_alt, docs);
    }
    embed_bwd(ids, dh_cur, g + c->p_embed, opt ? g + c->p_pos : nullptr, m.T, m.d, m.V, a.pad_token_id, m.S,
              opt ? OPT_POS_OFFSET : 0, s); ++n;
    go.exchange(0, c->n_zero_prefix);
  } catch (...) {
    gemm_set_sm_reserve(0);
    throw;
  }
  gemm_set_sm_reserve(0);
}

void ensure_ids(b200w_ctx* c, size_t n_tok) {
  if (c->ids_cap < n_tok) {
    if (c->ids_dev) {  // every kernel that read the old buffers was enqueued before this point
      B200W_CUDA(cudaStreamSynchronize(c->stream));
      c->release(c->ids_dev);
      c->release(c->labels_dev);
    }
    c->ids_dev = c->alloc<int32_t>(n_tok);
    c->labels_dev = c->alloc<int32_t>(n_tok);
    c->ids_cap = n_tok;
  }
  if (c->pinned_cap < 2 * n_tok) {
    if (c->pinned) {
      B200W_CUDA(cudaStreamSynchronize(c->stream));
      cudaFreeHost(c->pinned);
      c->pinned = nullptr;
    }
    B200W_CUDA(cudaMallocHost(reinterpret_cast<void**>(&c->pinned), 2 * n_tok * sizeof(int32_t)));
    c->pinned_cap = 2 * n_tok;
  }
}

// HF Trainer's num_items_in_batch (transformers 5.5 trainer.py:2136): labels != -100 counted on the
// UNSHIFTED labels of the whole batch, although the loss sums over the shifted ones (a row's first
// label never contributes a term but is counted). Round 1 counted the shifted labels, which is what
// model(input_ids, labels) does without a Trainer; the two differ by (S-1)/S on packed rows.
long count_valid(const int32_t* labels, int n_seqs, int S) {
  long nvalid = 0;
  const size_t n = static_cast<size_t>(n_seqs) * S;
  for (size_t i = 0; i < n; ++i) nvalid += labels[i] != -100;
  return nvalid;
}

void upload_batch(b200w_ctx* c, const int32_t* ids, const int32_t* labels, size_t n_tok) {
  // nn.Embedding / cross_entropy raise on out-of-range indices; here that would be a device trap
  // that poisons the CUDA context, so reject bad batches on the host (n_tok integer compares)
  const int32_t V = c->arch.vocab_size;
  for (size_t i = 0; i < n_tok; ++i) {
    if (ids[i] < 0 || ids[i] >= V) throw Error("check failed: token id outside the vocabulary");
    if (labels[i] != -100 && (labels[i] < 0 || labels[i] >= V))
      throw Error("check failed: label outside the vocabulary (use -100 to ignore)");
  }
  ensure_ids(c, n_tok);
  memcpy(c->pinned, ids, n_tok * sizeof(int32_t));
  memcpy(c->pinned + n_tok, labels, n_tok * sizeof(int32_t));
  B200W_CUDA(cudaMemcpyAsync(c->ids_dev, c->pinned, n_tok * sizeof(int32_t), cudaMemcpyHostToDevice,
                             c->stream));
  B200W_CUDA(cudaMemcpyAsync(c->labels_dev, c->pinned + n_tok, n_tok * sizeof(int32_t),
                             cudaMemcpyHostToDevice, c->stream));
}

// Per-document attention is built for the Llama family only: OPT's learned positions and Falcon's path take no
// positions. Checked before any GPU work.
void check_docs_family(const b200w_ctx* c) {
  B200W_CHECK(!is_opt(c->arch) && !is_falcon(c->arch),
              "per-document attention (positions) is built for the Llama family only");
}

// positions: HOST int32 [n_seqs, S] with HF position_ids semantics (DataCollatorWithFlattening): every row starts
// at 0 and each later entry is 0 (a new document) or the previous entry + 1, hence < S. Uploaded, and the
// DocBounds of the whole batch derived from them on the device.
void upload_positions(b200w_ctx* c, const int32_t* positions, int n_seqs) {
  const int S = c->arch.max_seq_len;
  for (int r = 0; r < n_seqs; ++r) {
    const int32_t* p = positions + static_cast<size_t>(r) * S;
    if (p[0] != 0) throw Error("check failed: positions of row " + std::to_string(r) + " do not start at 0");
    for (int i = 1; i < S; ++i)
      if (p[i] != 0 && p[i] != p[i - 1] + 1)
        throw Error("check failed: positions[" + std::to_string(r) + "][" + std::to_string(i) + "] = " +
                    std::to_string(p[i]) + " is neither 0 (a new document) nor the previous position + 1");
  }
  const size_t n = static_cast<size_t>(n_seqs) * S;
  if (c->docs_cap < n) {
    if (c->pos_dev) {  // every kernel that read the old buffers was enqueued before this point
      B200W_CUDA(cudaStreamSynchronize(c->stream));
      c->release(c->pos_dev);
      c->release(c->doc_start);
      c->release(c->doc_end);
    }
    c->pos_dev = c->alloc<int32_t>(n);
    c->doc_start = c->alloc<int32_t>(n);
    c->doc_end = c->alloc<int32_t>(n);
    c->docs_cap = n;
  }
  // pageable source: the call returns once the bytes are staged, so the caller's array may go
  B200W_CUDA(cudaMemcpyAsync(c->pos_dev, positions, n * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
  doc_bounds(c->pos_dev, c->doc_start, c->doc_end, static_cast<int>(n), S, c->stream); ++c->launches;
}

// the DocBounds of the rows [row0, ...) of the uploaded batch
DocBounds docs_at(const b200w_ctx* c, size_t row0) {
  const size_t off = row0 * c->arch.max_seq_len;
  return DocBounds{c->pos_dev + off, c->doc_start + off, c->doc_end + off};
}

// the loss normaliser of a target count taken on this process alone: cnt_dev = nvalid, inv_n = 1 / nvalid
void set_count(b200w_ctx* c, long nvalid) {
  set_count_kernel<<<1, 1, 0, c->stream>>>(c->cnt_dev, nvalid);
  inv_count_kernel<<<1, 1, 0, c->stream>>>(c->cnt_dev, c->inv_n);
  B200W_CUDA(cudaGetLastError());
}

// HF Trainer under DDP (transformers 5.5 trainer.py:2140-2143, average_tokens_across_devices = True,
// the TrainingArguments default): num_items_in_batch is gathered and SUMMED over the ranks, each
// rank's loss is sum(nll_r) / n_global * world (trainer.py:2013-2018) and DDP's mean removes the
// factor again, so the gradient is that of sum(nll over all ranks) / n_global -- the same number a
// single process computes on the global batch. Per-rank normalisation would differ whenever the
// ranks hold different numbers of target tokens (prompt-masked rows).
// The count never visits the host: it is summed by NCCL on the comm stream and its reciprocal lands
// in the device scalar c->inv_n that the loss kernels read (round 1 synchronised the host on this
// 8-byte all-reduce every step).
void set_global_count(b200w_ctx* c, long nvalid_local) {
  if (!c->comm) {
    set_count(c, nvalid_local);
    c->launches += 2;
    return;
  }
  cudaStream_t cs = c->comm_stream;
  // c->inv_n is still read by whatever the main stream has queued (the previous step's loss kernels)
  B200W_CUDA(cudaEventRecord(c->ev_grad, c->stream));
  B200W_CUDA(cudaStreamWaitEvent(cs, c->ev_grad, 0));
  set_count_kernel<<<1, 1, 0, cs>>>(c->cnt_dev, nvalid_local);
  B200W_CUDA(cudaGetLastError());
  B200W_NCCL(nccl().AllReduce(c->cnt_dev, c->cnt_dev, 1, kNcclInt64, kNcclSum, c->comm, cs));
  inv_count_kernel<<<1, 1, 0, cs>>>(c->cnt_dev, c->inv_n);
  B200W_CUDA(cudaGetLastError());
  B200W_CUDA(cudaEventRecord(c->ev_comm, cs));
  B200W_CUDA(cudaStreamWaitEvent(c->stream, c->ev_comm, 0));
  c->launches += 3;
}

// forward + loss + backward over a batch that is already on the device. nvalid = this rank's count
// of target tokens; with a communicator the gradients returned are those of the GLOBAL batch
// (sum over ranks of sum(nll) / n_global), all-reduced into the bf16 wire copy c->gw, and scal[0] is
// the global loss. docs: the batch's positions were uploaded (upload_positions): per-document attention.
void fwd_bwd_device(b200w_ctx* c, const int32_t* ids_dev, const int32_t* labels_dev, int n_seqs,
                    long nvalid, bool allow_overlap, bool docs = false) {
  const int S = c->arch.max_seq_len, mb = c->micro_batch;
  B200W_CHECK(c->has_model && c->training, "model not initialised for training");
  B200W_CHECK(n_seqs > 0 && n_seqs % mb == 0, "n_seqs must be a positive multiple of micro_batch");
  B200W_CHECK(nvalid >= 0, "negative target count");
  B200W_CHECK(c->comm || nvalid > 0, "batch has no valid target token");
  if (c->comm) ensure_wire(c);
  set_global_count(c, nvalid);
  allow_overlap = allow_overlap && ar_mode() != ArMode::End;
  B200W_CUDA(cudaMemsetAsync(c->scal, 0, 8 * sizeof(float), c->stream));
  B200W_CUDA(cudaMemsetAsync(c->g, 0, c->n_zero_prefix * sizeof(float), c->stream));
  const int n_micro = n_seqs / mb;
  for (int mi = 0; mi < n_micro; ++mi) {
    const int32_t* mids = ids_dev + static_cast<size_t>(mi) * mb * S;
    const int32_t* mlab = labels_dev + static_cast<size_t>(mi) * mb * S;
    const DocBounds db = docs ? docs_at(c, static_cast<size_t>(mi) * mb) : DocBounds{};
    const DocBounds* mdocs = docs ? &db : nullptr;
    {
      NvtxRange r("b200w forward");
      forward_micro(c, mids, mb, mdocs);
    }
    {
      NvtxRange r("b200w loss");
      loss_micro(c, mlab, mb);
    }
    const bool ar = allow_overlap && c->comm && mi == n_micro - 1;
    NvtxRange r(ar ? "b200w backward + gradient exchange" : "b200w backward");
    backward_micro(c, mids, mb, mi == 0, ar, mdocs);
  }
  if (c->comm) {
    if (!allow_overlap) allreduce_range(c, 0, c->n_elems);
    // the logged loss is the global token mean: sum the per-rank partials sum(nll_r) / n_global.
    // (comm_stream already waits for the end of the backward: the last allreduce_range did that)
    B200W_NCCL(nccl().AllReduce(c->scal, c->scal, 1, kNcclFloat32, kNcclSum, c->comm, c->comm_stream));
    ++c->launches;
    B200W_CUDA(cudaEventRecord(c->ev_comm, c->comm_stream));
    B200W_CUDA(cudaStreamWaitEvent(c->stream, c->ev_comm, 0));
  }
}

// positions (nullable): HOST [n_seqs, S], per-document attention (upload_positions)
void fwd_bwd_all(b200w_ctx* c, const int32_t* ids, const int32_t* labels, int n_seqs,
                 bool allow_overlap, const int32_t* positions = nullptr) {
  const int S = c->arch.max_seq_len;
  B200W_CHECK(c->has_model && c->training, "model not initialised for training");
  B200W_CHECK(n_seqs > 0, "empty batch");
  if (positions) check_docs_family(c);
  const long nvalid = count_valid(labels, n_seqs, S);
  upload_batch(c, ids, labels, static_cast<size_t>(n_seqs) * S);
  if (positions) upload_positions(c, positions, n_seqs);
  fwd_bwd_device(c, c->ids_dev, c->labels_dev, n_seqs, nvalid, allow_overlap, positions != nullptr);
}

// all-reduce is complete on c->stream; global-norm clip + AdamW over the flat parameter space.
// Gradient source: the fp32 accumulation buffer, or with a communicator the reduced bf16 wire copy.
void optimizer_step(b200w_ctx* c, float lr) {
  NvtxRange nvtx_range("b200w clip + AdamW");
  cudaStream_t s = c->stream;
  const bool wire = c->comm != nullptr;
  B200W_CUDA(cudaMemsetAsync(c->sumsq, 0, sizeof(double), s));
  c->step += 1;
  if (c->shard) {
    // each rank: sum of squares over its slices -> all-reduce of the scalar -> clip coefficient (identical on
    // every rank) -> AdamW on the owned slices -> all-gather of the bf16 compute copy, range by range
    const int N = c->nranks, r = c->rank;
    for (const auto& rg : c->ranges) {
      const size_t n = rg.cnt / N;
      grad_sumsq(c->gw + rg.off + r * n, true, n, c->sumsq, s); ++c->launches;
    }
    B200W_CUDA(cudaEventRecord(c->ev_grad, s));
    B200W_CUDA(cudaStreamWaitEvent(c->comm_stream, c->ev_grad, 0));
    B200W_NCCL(nccl().AllReduce(c->sumsq, c->sumsq, 1, kNcclFloat64, kNcclSum, c->comm, c->comm_stream));
    B200W_CUDA(cudaEventRecord(c->ev_comm, c->comm_stream));
    B200W_CUDA(cudaStreamWaitEvent(s, c->ev_comm, 0));
    clip_coef(c->sumsq, c->hp.max_grad_norm, 1.f, c->scal + 1, c->scal + 2, s); c->launches += 2;
    for (const auto& rg : c->ranges) {
      const size_t n = rg.cnt / N, lo = rg.off + r * n, co = rg.off / N;
      adamw_step(c->master + co, c->m + co, c->v + co, c->gw + lo, true, c->w + lo, n, lr, c->hp.beta1, c->hp.beta2,
                 c->hp.eps, rg.decay ? c->hp.weight_decay : 0.f, c->step, c->scal + 1, s);
      ++c->launches;
    }
    B200W_CUDA(cudaEventRecord(c->ev_grad, s));
    B200W_CUDA(cudaStreamWaitEvent(c->comm_stream, c->ev_grad, 0));
    for (const auto& rg : c->ranges) {
      const size_t n = rg.cnt / N;
      B200W_NCCL(nccl().AllGather(c->w + rg.off + r * n, c->w + rg.off, n, kNcclBfloat16, c->comm, c->comm_stream));
      ++c->launches;
    }
    B200W_CUDA(cudaEventRecord(c->ev_comm, c->comm_stream));
    B200W_CUDA(cudaStreamWaitEvent(s, c->ev_comm, 0));
    return;
  }
  const void* gsrc = wire ? static_cast<const void*>(c->gw) : static_cast<const void*>(c->g);
  grad_sumsq(gsrc, wire, c->n_elems, c->sumsq, s); ++c->launches;
  // the all-reduce summed per-rank partials that were already divided by the GLOBAL target count
  // (fwd_bwd_device), which is HF's DDP result: no 1/nranks here
  clip_coef(c->sumsq, c->hp.max_grad_norm, 1.f, c->scal + 1, c->scal + 2, s); ++c->launches;
  auto run = [&](size_t off, size_t n, float wd) {
    const void* gp = wire ? static_cast<const void*>(c->gw + off) : static_cast<const void*>(c->g + off);
    adamw_step(c->master + off, c->m + off, c->v + off, gp, wire, c->w + off, n, lr, c->hp.beta1,
               c->hp.beta2, c->hp.eps, wd, c->step, c->scal + 1, s);
    ++c->launches;
  };
  if (c->hp.weight_decay == 0.f) {
    run(0, c->n_elems, 0.f);
  } else {
    // HF Trainer's parameter groups (trainer.py get_decay_parameter_names): norm weights, LayerNorm
    // parameters and biases are not decayed
    for (const auto& sg : c->segs) run(sg.off, sg.n, sg.decay ? c->hp.weight_decay : 0.f);
  }
}

// sharded state: the owned part [lo, lo + n) of parameter p and where it sits in the packed master / m / v
struct OwnedPart { size_t lo, n, compact; };
bool owned_part(const b200w_ctx* c, const Param& p, OwnedPart* out) {
  for (const auto& rg : c->ranges) {
    if (p.off < rg.off || p.off >= rg.off + rg.cnt) continue;
    const size_t n = rg.cnt / c->nranks, s_lo = rg.off + c->rank * n, s_hi = s_lo + n;
    const size_t lo = std::max(s_lo, p.off), hi = std::min(s_hi, p.off + p.isize());
    if (lo >= hi) return false;
    *out = {lo, hi - lo, rg.off / c->nranks + (lo - s_lo)};
    return true;
  }
  return false;
}

// loss and grad-norm (each nullable) from the device scalars, once the main stream has drained
void read_scalars(b200w_ctx* ctx, float* loss_out, float* gnorm_out) {
  B200W_CUDA(cudaMemcpyAsync(ctx->host_scal, ctx->scal, 4 * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  B200W_CUDA(cudaStreamSynchronize(ctx->stream));
  if (loss_out) *loss_out = ctx->host_scal[0];
  if (gnorm_out) *gnorm_out = ctx->host_scal[2];
}

// The bodies of b200w_forward_backward, b200w_train_step and b200w_forward. positions (nullable, HOST
// [n_seqs, S]): per-document attention, the _docs forms.
void forward_backward_call(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels, const int32_t* positions,
                           int n_seqs, float* loss_out) {
  B200W_CHECK(ids && labels, "NULL batch");
  fwd_bwd_all(ctx, ids, labels, n_seqs, /*allow_overlap=*/false, positions);
  // the reduced gradients live in the bf16 wire copy: widen them for b200w_read_state(kind = 1)
  if (ctx->comm && !ctx->shard) { cast_bf16_to_f32(ctx->gw, ctx->g, ctx->n_elems, ctx->stream); ++ctx->launches; }
  read_scalars(ctx, loss_out, nullptr);
}

void train_step_call(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels, const int32_t* positions,
                     int n_seqs, float lr, float* loss_out, float* gnorm_out) {
  B200W_CHECK(ids && labels, "NULL batch");
  fwd_bwd_all(ctx, ids, labels, n_seqs, /*allow_overlap=*/true, positions);
  optimizer_step(ctx, lr);
  read_scalars(ctx, loss_out, gnorm_out);
}

void forward_call(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels, const int32_t* positions, int n_seqs,
                  float* logits_out, float* nll_out, float* loss_out) {
  B200W_CHECK(ctx->has_model && ids, "no model / NULL ids");
  B200W_CHECK(n_seqs >= 1 && n_seqs <= ctx->micro_batch, "n_seqs must be <= micro_batch");
  if (positions) check_docs_family(ctx);
  const int S = ctx->arch.max_seq_len, V = ctx->arch.vocab_size;
  const size_t T = static_cast<size_t>(n_seqs) * S;
  std::vector<int32_t> dummy;
  if (!labels) { dummy.assign(T, -100); }
  upload_batch(ctx, ids, labels ? labels : dummy.data(), T);
  DocBounds db{};
  if (positions) {
    upload_positions(ctx, positions, n_seqs);
    db = docs_at(ctx, 0);
  }
  forward_micro(ctx, ctx->ids_dev, n_seqs, positions ? &db : nullptr);
  if (logits_out) {
    void* scratch = nullptr;
    B200W_CUDA(cudaMalloc(&scratch, T * V * 4));
    cast_bf16_to_f32(ctx->logits, static_cast<float*>(scratch), T * V, ctx->stream);
    B200W_CUDA(cudaStreamSynchronize(ctx->stream));
    B200W_CUDA(cudaMemcpy(logits_out, scratch, T * V * 4, cudaMemcpyDeviceToHost));
    cudaFree(scratch);
  }
  if (labels && (nll_out || loss_out)) {
    set_count(ctx, count_valid(labels, n_seqs, S));
    B200W_CUDA(cudaMemsetAsync(ctx->scal, 0, 8 * sizeof(float), ctx->stream));
    loss_micro(ctx, ctx->labels_dev, n_seqs);
    read_scalars(ctx, loss_out, nullptr);
    if (nll_out) B200W_CUDA(cudaMemcpy(nll_out, ctx->nll, T * 4, cudaMemcpyDeviceToHost));
  }
  B200W_CUDA(cudaStreamSynchronize(ctx->stream));
}

}  // namespace

// ---- ctx_access.h ----------------------------------------------------------------------------
int ctx_device(b200w_ctx* c) { return c->device; }
cudaStream_t ctx_stream(b200w_ctx* c) { return c->stream; }
void ctx_set_error(b200w_ctx* c, const char* msg) { c->err = msg ? msg : ""; }
int64_t& ctx_launches(b200w_ctx* c) { return c->launches; }
void* ctx_infer_slot(b200w_ctx* c) { return c->infer; }
void ctx_set_infer(b200w_ctx* c, void* p, void (*destroy)(void*)) {
  c->infer = p;
  c->infer_destroy = destroy;
}
void ctx_fill_normal(b200w_ctx* c, void* w_bf16, size_t n, uint64_t seed, float std) {
  init_normal_kernel<<<sm_count() * 8, 256, 0, c->stream>>>(nullptr, static_cast<bf16*>(w_bf16), n, seed, std);
  B200W_CUDA(cudaGetLastError());
}
void ctx_fill_const(b200w_ctx* c, void* w_bf16, size_t n, float value) {
  fill_kernel<<<64, 256, 0, c->stream>>>(nullptr, static_cast<bf16*>(w_bf16), n, value);
  B200W_CUDA(cudaGetLastError());
}

// ============================================================================================
// C ABI
// ============================================================================================
extern "C" {

int b200w_abi_version(void) { return B200W_ABI_VERSION; }
int b200w_debug_gemm_raster(int M, int N, int K, int tile_m, int tile_n, int32_t* coords) {
  if (M <= 0 || N <= 0 || K <= 0 || tile_m <= 0 || tile_n <= 0) return -1;
  return b200w::gemm_debug_raster(M, N, K, tile_m, tile_n, coords);
}

int b200w_create(int device, b200w_ctx** out) {
  if (!out) return B200W_ERR_INVALID;
  *out = nullptr;
  try {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || device < 0 || device >= count) {
      cudaGetLastError();
      g_create_error = "no usable CUDA device " + std::to_string(device) +
                       " (b200w has no CPU fallback): " + cudaGetErrorString(e);
      return B200W_ERR_CUDA;
    }
    B200W_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    B200W_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
      g_create_error = std::string("b200w is built for sm_90a only; device is ") + prop.name;
      return B200W_ERR_CUDA;
    }
    auto c = std::make_unique<b200w_ctx>();
    c->device = device;
    B200W_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    B200W_CUDA(cudaStreamCreateWithFlags(&c->comm_stream, cudaStreamNonBlocking));
    B200W_CUDA(cudaEventCreateWithFlags(&c->ev_grad, cudaEventDisableTiming));
    B200W_CUDA(cudaEventCreateWithFlags(&c->ev_comm, cudaEventDisableTiming));
    B200W_CUDA(cudaMallocHost(reinterpret_cast<void**>(&c->host_scal), 8 * sizeof(float)));
    *out = c.release();
    return B200W_OK;
  } catch (const std::exception& e) {
    g_create_error = e.what();
    return B200W_ERR_CUDA;
  }
}

void b200w_destroy(b200w_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  // After a device fault (e.g. the bounded mbarrier wait trapped) or an NCCL error, waiting for the
  // device or for a clean communicator shutdown can block for ever: peers are still inside a
  // collective that will never complete. Abort instead, so that this process can exit and the
  // launcher can tear the job down (a rank that fails but does not exit keeps its peers spinning
  // inside the collective).
  const bool dead = ctx->poisoned || cudaDeviceSynchronize() != cudaSuccess;
  if (ctx->comm) {
    if (!dead) nccl().CommDestroy(ctx->comm);
    else if (nccl().CommAbort) nccl().CommAbort(ctx->comm);
  }
  if (ctx->infer && ctx->infer_destroy) ctx->infer_destroy(ctx->infer);
  ctx->free_all();
  if (ctx->pinned) cudaFreeHost(ctx->pinned);
  if (ctx->host_scal) cudaFreeHost(ctx->host_scal);
  if (ctx->ev_grad) cudaEventDestroy(ctx->ev_grad);
  if (ctx->ev_comm) cudaEventDestroy(ctx->ev_comm);
  if (ctx->ev_t0) cudaEventDestroy(ctx->ev_t0);
  if (ctx->ev_t1) cudaEventDestroy(ctx->ev_t1);
  for (cudaEvent_t e : ctx->prof_events) cudaEventDestroy(e);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  if (ctx->comm_stream) cudaStreamDestroy(ctx->comm_stream);
  delete ctx;
}

const char* b200w_last_error(const b200w_ctx* ctx) {
  return ctx ? ctx->err.c_str() : g_create_error.c_str();
}

int b200w_sync(b200w_ctx* ctx) {
  return guarded(ctx, [&] {
    B200W_CUDA(cudaStreamSynchronize(ctx->stream));
    B200W_CUDA(cudaStreamSynchronize(ctx->comm_stream));
  });
}

void b200w_default_hparams(b200w_hparams* hp) {
  if (!hp) return;
  hp->lr = 5e-5f; hp->beta1 = 0.9f; hp->beta2 = 0.999f; hp->eps = 1e-8f;
  hp->weight_decay = 0.0f; hp->max_grad_norm = 1.0f;
}

int b200w_model_init(b200w_ctx* ctx, const b200w_arch* arch, const b200w_hparams* hp,
                     int micro_batch, int training) {
  return guarded(ctx, [&] {
    B200W_CHECK(arch != nullptr, "arch is NULL");
    B200W_CHECK(!ctx->has_model, "model already initialised");
    B200W_CHECK(arch->family == B200W_FAMILY_LLAMA || arch->family == B200W_FAMILY_OPT ||
                    arch->family == B200W_FAMILY_FALCON,
                "the fine-tune engine builds the Llama, OPT and Falcon families");
    const bool opt = arch->family == B200W_FAMILY_OPT, falcon = arch->family == B200W_FAMILY_FALCON;
    if (falcon) {
      B200W_CHECK(arch->head_dim == 64 || arch->head_dim == 128, "Falcon: head_dim must be 64 or 128");
      B200W_CHECK(arch->hidden_size == arch->num_heads * arch->head_dim, "Falcon: hidden_size = heads x head_dim");
    } else if (opt) {
      B200W_CHECK(arch->head_dim == 64 || arch->head_dim == 128, "OPT: head_dim must be 64 or 128");
      B200W_CHECK(arch->num_kv_heads == arch->num_heads, "OPT has no grouped-query attention");
      B200W_CHECK(arch->hidden_size == arch->num_heads * arch->head_dim, "OPT: hidden_size = heads x head_dim");
      B200W_CHECK(arch->max_positions >= arch->max_seq_len,
                  "OPT: max_seq_len exceeds the learned position table (max_position_embeddings)");
    } else {
      B200W_CHECK(arch->head_dim == 128, "Llama: head_dim must be 128");
    }
    B200W_CHECK(arch->num_heads % arch->num_kv_heads == 0, "heads must be a multiple of kv heads");
    B200W_CHECK(arch->hidden_size % 8 == 0 && arch->intermediate_size % 8 == 0 &&
                    arch->vocab_size % 8 == 0,
                "sizes must be multiples of 8");
    B200W_CHECK(arch->max_seq_len % 128 == 0, "max_seq_len must be a multiple of 128");
    B200W_CHECK(arch->pad_token_id >= -1 && arch->pad_token_id < arch->vocab_size, "bad pad_token_id");
    B200W_CHECK(micro_batch >= 1, "micro_batch must be >= 1");
    ctx->arch = *arch;
    if (hp) ctx->hp = *hp; else b200w_default_hparams(&ctx->hp);
    ctx->micro_batch = micro_batch;
    B200W_CHECK(training >= 0 && (training & ~B200W_TRAIN_RECOMPUTE) <= 2, "training: 0, 1 or 2, optionally | B200W_TRAIN_RECOMPUTE");
    const bool recompute = (training & B200W_TRAIN_RECOMPUTE) != 0;
    training &= ~B200W_TRAIN_RECOMPUTE;
    B200W_CHECK(!recompute || (training != 0 && !opt && !falcon),
                "activation recomputation is built for fine-tuning the Llama family");
    ctx->training = training != 0;
    ctx->shard = training == 2;
    ctx->recompute = recompute;
    B200W_CHECK(!(training == 2 && arch->head_dim != 128), "sharded optimiser state is built for head_dim 128 models");
    B200W_CHECK(!ctx->shard || (ctx->comm && ctx->nranks > 1),
                "sharded optimiser state needs the communicator first: b200w_comm_init before b200w_model_init(training = 2)");
    ctx->dhp = 128;
    if (opt) build_params_opt(ctx); else if (falcon) build_params_falcon(ctx); else build_params_llama(ctx);
    build_segments(ctx);
    {
      const size_t d = arch->hidden_size, f = arch->intermediate_size, V = arch->vocab_size;
      const size_t qd = qd_of(ctx), qkvd = qkv_dim(ctx);
      std::vector<std::pair<size_t, size_t>> mats;
      for (const auto& lp : ctx->lp) {
        mats.push_back({lp.wqkv, qkvd * d});
        mats.push_back({lp.wo, d * qd});
        mats.push_back({lp.wgu, (gated_mlp(ctx->arch) ? 2 * f : f) * d});
        mats.push_back({lp.wd, d * f});
      }
      if (!tied_head(ctx)) mats.push_back({ctx->p_lm, V * d});
      build_ranges(ctx, mats);
      size_t covered = 0;
      for (const auto& rg : ctx->ranges) {
        B200W_CHECK(rg.off == covered, "internal: exchange ranges do not tile the parameter space");
        covered += rg.cnt;
        if (ctx->shard)
          B200W_CHECK(rg.cnt % (8 * static_cast<size_t>(ctx->nranks)) == 0,
                      "sharded state: every matrix must split into nranks slices of a multiple of 8 elements");
      }
      B200W_CHECK(covered == ctx->n_elems, "internal: exchange ranges do not cover the parameter space");
    }
    ctx->w = ctx->alloc<bf16>(ctx->n_elems);
    B200W_CUDA(cudaMemsetAsync(ctx->w, 0, ctx->n_elems * sizeof(bf16), ctx->stream));  // head padding = 0
    if (ctx->training) {
      // replicated: fp32 master + Adam moments for every parameter; sharded: for this rank's 1/nranks only
      const size_t n_state = ctx->shard ? ctx->n_elems / ctx->nranks : ctx->n_elems;
      ctx->master = ctx->alloc<float>(n_state);
      ctx->m = ctx->alloc<float>(n_state);
      ctx->v = ctx->alloc<float>(n_state);
      ctx->g = ctx->alloc<float>(ctx->n_elems);
      B200W_CUDA(cudaMemsetAsync(ctx->master, 0, n_state * sizeof(float), ctx->stream));
      B200W_CUDA(cudaMemsetAsync(ctx->m, 0, n_state * sizeof(float), ctx->stream));
      B200W_CUDA(cudaMemsetAsync(ctx->v, 0, n_state * sizeof(float), ctx->stream));
      B200W_CUDA(cudaMemsetAsync(ctx->g, 0, ctx->n_elems * sizeof(float), ctx->stream));
    }
    alloc_activations(ctx);
    B200W_CUDA(cudaStreamSynchronize(ctx->stream));
    ctx->has_model = true;
    ctx->step = 0;
  });
}

int b200w_param_count(b200w_ctx* ctx, int64_t* n_tensors, int64_t* n_elements) {
  return guarded(ctx, [&] {
    B200W_CHECK(ctx->has_model, "no model");
    if (n_tensors) *n_tensors = static_cast<int64_t>(ctx->params.size());
    if (n_elements) *n_elements = static_cast<int64_t>(ctx->n_elems);
  });
}

int b200w_param_info(b200w_ctx* ctx, int64_t index, char* name, size_t name_cap, int64_t* rows,
                     int64_t* cols) {
  return guarded(ctx, [&] {
    B200W_CHECK(ctx->has_model && index >= 0 && index < (int64_t)ctx->params.size(), "bad index");
    const Param& p = ctx->params[index];
    if (name && name_cap) {
      strncpy(name, p.name.c_str(), name_cap - 1);
      name[name_cap - 1] = 0;
    }
    if (rows) *rows = p.rows;
    if (cols) *cols = p.cols;
  });
}

static const Param& find_param(b200w_ctx* ctx, const char* name, int64_t n_elements) {
  B200W_CHECK(ctx->has_model && name, "no model / name");
  auto it = ctx->index.find(name);
  if (it == ctx->index.end()) throw Error(std::string("check failed: unknown parameter ") + name);
  const Param& p = ctx->params[it->second];
  B200W_CHECK(n_elements == p.rows * p.cols, "element count does not match the parameter shape");
  return p;
}

// dense host tensor -> the parameter's (possibly head-padded) place in master / w
int b200w_load_tensor(b200w_ctx* ctx, const char* name, const void* host, b200w_dtype dtype,
                      int64_t n_elements) {
  return guarded(ctx, [&] {
    const Param& p = find_param(ctx, name, n_elements);
    B200W_CHECK(host && (dtype == B200W_BF16 || dtype == B200W_F32), "bad host buffer / dtype");
    const size_t n = static_cast<size_t>(n_elements);
    cudaStream_t s = ctx->stream;
    if (ctx->shard) {
      // every rank holds the whole bf16 compute copy; the fp32 master exists for the owned slice only and
      // receives the exact fp32 values of an fp32 checkpoint there
      float* dense = nullptr;
      void* raw = nullptr;
      B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&dense), n * 4));
      try {
        if (dtype == B200W_F32) {
          B200W_CUDA(cudaMemcpyAsync(dense, host, n * 4, cudaMemcpyHostToDevice, s));
          cast_f32_to_bf16(dense, ctx->w + p.off, n, s);
        } else {
          B200W_CUDA(cudaMemcpyAsync(ctx->w + p.off, host, n * 2, cudaMemcpyHostToDevice, s));
          cast_bf16_to_f32(ctx->w + p.off, dense, n, s);
        }
        OwnedPart op;
        if (owned_part(ctx, p, &op))
          B200W_CUDA(cudaMemcpyAsync(ctx->master + op.compact, dense + (op.lo - p.off), op.n * 4,
                                     cudaMemcpyDeviceToDevice, s));
        B200W_CUDA(cudaStreamSynchronize(s));
      } catch (...) { cudaFree(dense); cudaFree(raw); throw; }
      cudaFree(dense);
      return;
    }
    if (p.pad == 0) {
      if (dtype == B200W_F32) {
        float* tmp = ctx->training ? ctx->master + p.off : nullptr;
        void* scratch = nullptr;
        if (!tmp) { B200W_CUDA(cudaMalloc(&scratch, n * 4)); tmp = static_cast<float*>(scratch); }
        B200W_CUDA(cudaMemcpyAsync(tmp, host, n * 4, cudaMemcpyHostToDevice, s));
        cast_f32_to_bf16(tmp, ctx->w + p.off, n, s);
        B200W_CUDA(cudaStreamSynchronize(s));
        if (scratch) cudaFree(scratch);
      } else {
        B200W_CUDA(cudaMemcpyAsync(ctx->w + p.off, host, n * 2, cudaMemcpyHostToDevice, s));
        if (ctx->training) cast_bf16_to_f32(ctx->w + p.off, ctx->master + p.off, n, s);
        B200W_CUDA(cudaStreamSynchronize(s));
      }
      return;
    }
    // head-padded parameter: stage dense fp32 on the device, scatter into the padded rows / columns
    float* dense = nullptr;
    void* raw = nullptr;
    B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&dense), n * 4));
    try {
      if (dtype == B200W_F32) {
        B200W_CUDA(cudaMemcpyAsync(dense, host, n * 4, cudaMemcpyHostToDevice, s));
      } else {
        B200W_CUDA(cudaMalloc(&raw, n * 2));
        B200W_CUDA(cudaMemcpyAsync(raw, host, n * 2, cudaMemcpyHostToDevice, s));
        cast_bf16_to_f32(raw, dense, n, s);
      }
      pad_scatter_kernel<<<sm_count() * 4, 256, 0, s>>>(dense, ctx->training ? ctx->master + p.off : nullptr,
                                                        ctx->w + p.off, p.rows, p.cols, p.icols, p.pad,
                                                        ctx->arch.head_dim, ctx->dhp);
      B200W_CUDA(cudaGetLastError());
      B200W_CUDA(cudaStreamSynchronize(s));
    } catch (...) { cudaFree(dense); cudaFree(raw); throw; }
    cudaFree(dense);
    cudaFree(raw);
  });
}

namespace {
// the parameter's dense HF-shaped values as fp32 on the host, from an fp32 state array (srcf) or the
// bf16 compute copy (srcb)
void read_dense(b200w_ctx* ctx, const Param& p, const float* srcf, const bf16* srcb, float* host) {
  const size_t n = static_cast<size_t>(p.rows) * p.cols;
  cudaStream_t s = ctx->stream;
  B200W_CUDA(cudaStreamSynchronize(s));
  if (p.pad == 0 && srcf) {
    B200W_CUDA(cudaMemcpy(host, srcf + p.off, n * 4, cudaMemcpyDeviceToHost));
    return;
  }
  float* dense = nullptr;
  B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&dense), n * 4));
  try {
    pad_gather_kernel<<<sm_count() * 4, 256, 0, s>>>(srcf ? srcf + p.off : nullptr, srcb ? srcb + p.off : nullptr,
                                                     dense, p.rows, p.cols, p.icols, p.pad, ctx->arch.head_dim,
                                                     ctx->dhp);
    B200W_CUDA(cudaGetLastError());
    B200W_CUDA(cudaStreamSynchronize(s));
    B200W_CUDA(cudaMemcpy(host, dense, n * 4, cudaMemcpyDeviceToHost));
  } catch (...) { cudaFree(dense); throw; }
  cudaFree(dense);
}
}  // namespace

int b200w_read_tensor(b200w_ctx* ctx, const char* name, void* host, b200w_dtype dtype,
                      int64_t n_elements) {
  return guarded(ctx, [&] {
    const Param& p = find_param(ctx, name, n_elements);
    B200W_CHECK(host && (dtype == B200W_BF16 || dtype == B200W_F32), "bad host buffer / dtype");
    const size_t n = static_cast<size_t>(n_elements);
    if (dtype == B200W_F32) {
      // fp32 master when this context holds all of it; with sharded state the (complete, all-gathered)
      // bf16 compute copy widened to fp32
      const bool full_master = ctx->training && !ctx->shard;
      read_dense(ctx, p, full_master ? ctx->master : nullptr, full_master ? nullptr : ctx->w,
                 static_cast<float*>(host));
      return;
    }
    B200W_CUDA(cudaStreamSynchronize(ctx->stream));
    if (p.pad == 0) {
      B200W_CUDA(cudaMemcpy(host, ctx->w + p.off, n * 2, cudaMemcpyDeviceToHost));
      return;
    }
    // padded + bf16: gather as fp32 (exact: the values are bf16), round back on the host side of the copy
    std::vector<float> tmp(n);
    read_dense(ctx, p, nullptr, ctx->w, tmp.data());
    uint16_t* out = static_cast<uint16_t*>(host);
    for (size_t i = 0; i < n; ++i) {
      uint32_t u;
      memcpy(&u, &tmp[i], 4);
      out[i] = static_cast<uint16_t>(u >> 16);  // exact: low 16 bits are zero
    }
  });
}

int b200w_read_state(b200w_ctx* ctx, const char* name, int kind, float* host, int64_t n_elements) {
  return guarded(ctx, [&] {
    const Param& p = find_param(ctx, name, n_elements);
    B200W_CHECK(ctx->training && host && kind >= 0 && kind <= 3, "bad kind / not training");
    if (ctx->shard) {
      // only 1/nranks of master / m / v lives here and the reduced gradient is scattered: the weights are
      // readable (from the all-gathered compute copy), the rest is not a single-rank quantity
      if (kind != 0) throw Error("check failed: optimiser state is sharded over the ranks (kind 1..3 unavailable)");
      read_dense(ctx, p, nullptr, ctx->w, host);
      return;
    }
    const float* src[4] = {ctx->master, ctx->g, ctx->m, ctx->v};
    read_dense(ctx, p, src[kind], nullptr, host);
  });
}

int b200w_init_random(b200w_ctx* ctx, uint64_t seed, float std) {
  return guarded(ctx, [&] {
    B200W_CHECK(ctx->has_model, "no model");
    for (const Param& p : ctx->params) {
      const size_t n = p.isize();
      if (ctx->shard) {   // whole bf16 copy + the owned slice of the master, from the same per-element stream
        OwnedPart op{};
        const bool own = owned_part(ctx, p, &op);
        if (p.is_norm || p.is_zero_init) {
          const float val = p.is_norm ? 1.0f : 0.0f;
          fill_kernel<<<64, 256, 0, ctx->stream>>>(nullptr, ctx->w + p.off, n, val);
          if (own) fill_kernel<<<64, 256, 0, ctx->stream>>>(ctx->master + op.compact, nullptr, op.n, val);
        } else {
          init_normal_kernel<<<sm_count() * 8, 256, 0, ctx->stream>>>(nullptr, ctx->w + p.off, n, seed + p.off, std);
          if (own)
            init_normal_kernel<<<sm_count() * 8, 256, 0, ctx->stream>>>(ctx->master + op.compact, nullptr, op.n,
                                                                        seed + p.off, std, op.lo - p.off);
        }
        continue;
      }
      float* mp = ctx->training ? ctx->master + p.off : nullptr;
      if (p.is_norm || p.is_zero_init)
        fill_kernel<<<64, 256, 0, ctx->stream>>>(mp, ctx->w + p.off, n, p.is_norm ? 1.0f : 0.0f);
      else
        init_normal_kernel<<<sm_count() * 8, 256, 0, ctx->stream>>>(mp, ctx->w + p.off, n,
                                                                    seed + p.off, std);
      if (p.pad)
        pad_zero_kernel<<<sm_count() * 4, 256, 0, ctx->stream>>>(mp, ctx->w + p.off, p.irows, p.icols, p.pad,
                                                                 ctx->arch.head_dim, ctx->dhp);
    }
    B200W_CUDA(cudaGetLastError());
    B200W_CUDA(cudaStreamSynchronize(ctx->stream));
  });
}

int b200w_comm_unique_id(void* id128) {
  if (!id128) return B200W_ERR_INVALID;
  try {
    int r = nccl().GetUniqueId(id128);
    if (r != 0) { g_create_error = nccl().GetErrorString(r); return B200W_ERR_NCCL; }
    return B200W_OK;
  } catch (const std::exception& e) {
    g_create_error = e.what();
    return B200W_ERR_NCCL;
  }
}

int b200w_comm_init(b200w_ctx* ctx, int rank, int nranks, const void* id128) {
  return guarded(ctx, [&] {
    B200W_CHECK(id128 && nranks >= 1 && rank >= 0 && rank < nranks, "bad rank / id");
    B200W_CHECK(!ctx->comm, "communicator already initialised");
    // The gradient all-reduce runs under the last backward. NCCL's CTAs and the persistent GEMM CTAs
    // (one per SM, ~200 KB of shared memory each) cannot share an SM, so the two are given disjoint
    // SM budgets: NCCL is capped at R CTAs (NCCL_MAX_CTAS, unless the user set it) and the GEMMs of
    // that backward launch on SMs - R. B200W_AR_SM_RESERVE overrides R (0: no partition).
    // R = 8: the whole 13.5 GB exchange has the last micro-step's backward to hide in, so even 8 CTAs are far
    // more bandwidth than it needs; every reserved SM costs the GEMMs of that backward 1/132 of an H100.
    int reserve = 8;
    if (const char* e = getenv("B200W_AR_SM_RESERVE")) reserve = atoi(e);
    if (reserve < 0 || reserve > 64) reserve = 8;
    ctx->ar_sm_reserve = nranks > 1 ? reserve : 0;
    if (reserve > 0) setenv("NCCL_MAX_CTAS", std::to_string(reserve).c_str(), /*overwrite=*/0);
    Uid uid;
    memcpy(&uid, id128, sizeof(uid));
    try {
      B200W_NCCL(nccl().CommInitRank(&ctx->comm, nranks, uid, rank));
    } catch (const Error& e) {
      throw NcclError(e.what());
    }
    ctx->rank = rank;
    ctx->nranks = nranks;
    // NCCL connects its transports lazily, at the first collective of each kind (for 8 ranks:
    // P2P rings plus NVLS multicast objects -- seconds of driver work). Do that now, with the
    // message classes the step uses (large bf16 sum, one int64, one float) and nothing else on the
    // GPU, instead of in the middle of the first backward.
    {
      const size_t n_big = size_t(64) << 20;  // 128 MB of bf16: same protocol/algorithm class as a matrix gradient
      bf16* scratch = nullptr;
      B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&scratch), n_big * sizeof(bf16)));
      cudaStream_t cs = ctx->comm_stream;
      try {
        B200W_CUDA(cudaMemsetAsync(scratch, 0, n_big * sizeof(bf16), cs));
        B200W_NCCL(nccl().AllReduce(scratch, scratch, n_big, kNcclBfloat16, kNcclSum, ctx->comm, cs));
        B200W_NCCL(nccl().AllReduce(scratch, scratch, 1, kNcclFloat32, kNcclSum, ctx->comm, cs));
        B200W_NCCL(nccl().AllReduce(scratch, scratch, 1, kNcclInt64, kNcclSum, ctx->comm, cs));
        B200W_CUDA(cudaStreamSynchronize(cs));
      } catch (...) {
        cudaFree(scratch);
        throw;
      }
      B200W_CUDA(cudaFree(scratch));
    }
  });
}

int b200w_forward_backward(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels, int n_seqs,
                           float* loss_out) {
  return guarded(ctx, [&] { forward_backward_call(ctx, ids, labels, nullptr, n_seqs, loss_out); });
}
int b200w_forward_backward_docs(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels, const int32_t* positions,
                                int n_seqs, float* loss_out) {
  return guarded(ctx, [&] {
    B200W_CHECK(positions, "NULL positions");
    forward_backward_call(ctx, ids, labels, positions, n_seqs, loss_out);
  });
}

int b200w_train_step(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels, int n_seqs, float lr,
                     float* loss_out, float* gnorm_out) {
  return guarded(ctx, [&] { train_step_call(ctx, ids, labels, nullptr, n_seqs, lr, loss_out, gnorm_out); });
}
int b200w_train_step_docs(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels, const int32_t* positions,
                          int n_seqs, float lr, float* loss_out, float* gnorm_out) {
  return guarded(ctx, [&] {
    B200W_CHECK(positions, "NULL positions");
    train_step_call(ctx, ids, labels, positions, n_seqs, lr, loss_out, gnorm_out);
  });
}

int b200w_train_step_resident(b200w_ctx* ctx, const int32_t* ids_dev, const int32_t* labels_dev,
                              int n_seqs, int64_t n_valid, float lr) {
  return guarded(ctx, [&] {
    B200W_CHECK(ids_dev && labels_dev, "NULL batch");
    fwd_bwd_device(ctx, ids_dev, labels_dev, n_seqs, static_cast<long>(n_valid), /*allow_overlap=*/true);
    optimizer_step(ctx, lr);
  });
}

int b200w_read_scalars(b200w_ctx* ctx, float* loss_out, float* gnorm_out) {
  return guarded(ctx, [&] {
    B200W_CHECK(ctx->has_model, "no model");
    read_scalars(ctx, loss_out, gnorm_out);
  });
}

int b200w_timer_start(b200w_ctx* ctx) {
  return guarded(ctx, [&] {
    if (!ctx->ev_t0) {
      B200W_CUDA(cudaEventCreate(&ctx->ev_t0));
      B200W_CUDA(cudaEventCreate(&ctx->ev_t1));
    }
    B200W_CUDA(cudaEventRecord(ctx->ev_t0, ctx->stream));
  });
}

int b200w_timer_stop(b200w_ctx* ctx, float* ms_out) {
  return guarded(ctx, [&] {
    B200W_CHECK(ctx->ev_t0 != nullptr && ms_out, "timer not started");
    // everything the step put on the comm stream has already been joined into ctx->stream
    B200W_CUDA(cudaEventRecord(ctx->ev_t1, ctx->stream));
    B200W_CUDA(cudaEventSynchronize(ctx->ev_t1));
    B200W_CUDA(cudaEventElapsedTime(ms_out, ctx->ev_t0, ctx->ev_t1));
  });
}

int b200w_profile_gemm(b200w_ctx* ctx, int enable) {
  return guarded(ctx, [&] {
    ctx->prof_gemm = enable != 0;
    if (enable) { ctx->prof_used = 0; ctx->prof_flops = 0; }
  });
}

int b200w_profile_read(b200w_ctx* ctx, double* ms_out, double* flops_out, int64_t* launches_out) {
  return guarded(ctx, [&] {
    B200W_CUDA(cudaStreamSynchronize(ctx->stream));
    double ms = 0;
    for (size_t i = 0; i + 1 < ctx->prof_used; i += 2) {
      float t = 0;
      B200W_CUDA(cudaEventElapsedTime(&t, ctx->prof_events[i], ctx->prof_events[i + 1]));
      ms += t;
    }
    if (ms_out) *ms_out = ms;
    if (flops_out) *flops_out = ctx->prof_flops;
    if (launches_out) *launches_out = static_cast<int64_t>(ctx->prof_used / 2);
  });
}

int b200w_forward(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels, int n_seqs,
                  float* logits_out, float* nll_out, float* loss_out) {
  return guarded(ctx, [&] { forward_call(ctx, ids, labels, nullptr, n_seqs, logits_out, nll_out, loss_out); });
}
int b200w_forward_docs(b200w_ctx* ctx, const int32_t* ids, const int32_t* labels, const int32_t* positions,
                       int n_seqs, float* logits_out, float* nll_out, float* loss_out) {
  return guarded(ctx, [&] {
    B200W_CHECK(positions, "NULL positions");
    forward_call(ctx, ids, labels, positions, n_seqs, logits_out, nll_out, loss_out);
  });
}

int64_t b200w_launch_count(const b200w_ctx* ctx) { return ctx ? ctx->launches : 0; }
int64_t b200w_device_bytes(const b200w_ctx* ctx) { return ctx ? ctx->dev_bytes : 0; }

// ---- per-kernel hooks ---------------------------------------------------------------------
#define HOOK(body)                                              \
  return guarded(ctx, [&] {                                     \
    body;                                                       \
    ++ctx->launches;                                            \
    B200W_CUDA(cudaStreamSynchronize(ctx->stream));             \
  })

int b200w_op_gemm(b200w_ctx* ctx, const void* A, int a_mn, int lda, const void* B, int b_mn, int ldb,
                  void* D, const void* C, int out_f32, int ldd, int M, int N, int K, int block_n) {
  HOOK(gemm_bf16(A, a_mn != 0, lda, B, b_mn != 0, ldb, D, C, out_f32 != 0, ldd, M, N, K, block_n,
                 ctx->stream));
}
int b200w_op_gemm_bias(b200w_ctx* ctx, const void* A, int lda, const void* B, int ldb, void* D, const void* C, int ldd,
                       int M, int N, int K, const void* bias, int act, int block_n) {
  HOOK(gemm_bf16_ex(A, false, lda, B, false, ldb, D, C, false, ldd, M, N, K, block_n, bias, act, ctx->stream));
}
int b200w_op_gemm_decode(b200w_ctx* ctx, const void* X, const void* W, void* out, const void* C, int M,
                         int N, int K, int split_k) {
  return guarded(ctx, [&] {
    float* ws = nullptr;
    unsigned* cnt = nullptr;
    if (split_k) {
      B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&ws), static_cast<size_t>(M) * N * 4));
      B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&cnt), ((N + 127) / 128) * 4));
      B200W_CUDA(cudaMemsetAsync(ws, 0, static_cast<size_t>(M) * N * 4, ctx->stream));
      B200W_CUDA(cudaMemsetAsync(cnt, 0, ((N + 127) / 128) * 4, ctx->stream));
    }
    try {
      gemm_decode(X, W, out, C, ws, cnt, M, N, K, N, 0, ctx->stream);
      gemm_decode(X, W, out, C, ws, cnt, M, N, K, N, 0, ctx->stream);  // twice: the scratch must come back clean
      ctx->launches += 2;
      B200W_CUDA(cudaStreamSynchronize(ctx->stream));
    } catch (...) { cudaFree(ws); cudaFree(cnt); throw; }
    cudaFree(ws);
    cudaFree(cnt);
  });
}
int b200w_op_embed_fwd(b200w_ctx* ctx, const int32_t* ids, const void* table, const void* pos_table,
                       void* out, int T, int d, int vocab, int S, int pos_offset) {
  HOOK(embed_fwd(ids, table, pos_table, out, T, d, vocab, S, pos_offset, ctx->stream));
}
int b200w_op_embed_bwd(b200w_ctx* ctx, const int32_t* ids, const void* dout, float* dtable, float* dpos,
                       int T, int d, int vocab, int pad_id, int S, int pos_offset) {
  HOOK(embed_bwd(ids, dout, dtable, dpos, T, d, vocab, pad_id, S, pos_offset, ctx->stream));
}
int b200w_op_layernorm_fwd(b200w_ctx* ctx, const void* x, const void* w, const void* b, void* y, float* mean,
                           float* rstd, int T, int d, float eps) {
  HOOK(layernorm_fwd(x, w, b, y, mean, rstd, T, d, eps, ctx->stream));
}
int b200w_op_layernorm_bwd(b200w_ctx* ctx, const void* dy, const void* x, const void* w, const float* mean,
                           const float* rstd, const void* dresid, void* dx, float* dw, float* db, int T,
                           int d) {
  return guarded(ctx, [&] {
    float* part = nullptr;
    B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&part),
                          static_cast<size_t>(rmsnorm_bwd_blocks(T)) * 2 * d * sizeof(float)));
    try {
      layernorm_bwd(dy, x, w, mean, rstd, dresid, dx, dw, db, part, T, d, ctx->stream);
      ctx->launches += 3;
      B200W_CUDA(cudaStreamSynchronize(ctx->stream));
    } catch (...) { cudaFree(part); throw; }
    cudaFree(part);
  });
}
int b200w_op_bias_act(b200w_ctx* ctx, void* x, const void* bias, int T, int N, int ld, int act) {
  HOOK(bias_act(x, bias, T, N, ld, act, ctx->stream));
}
int b200w_op_relu_bwd(b200w_ctx* ctx, const void* dy, const void* act, void* dz, int64_t n) {
  HOOK(relu_bwd(dy, act, dz, static_cast<size_t>(n), ctx->stream));
}
int b200w_op_gelu_fwd(b200w_ctx* ctx, const void* x, void* y, int64_t n) {
  HOOK(gelu_fwd(x, y, static_cast<size_t>(n), ctx->stream));
}
int b200w_op_gelu_bwd(b200w_ctx* ctx, const void* dy, const void* x, void* dx, int64_t n) {
  HOOK(gelu_bwd(dy, x, dx, static_cast<size_t>(n), ctx->stream));
}
int b200w_op_colsum(b200w_ctx* ctx, const void* dy, float* db, int T, int N, int ld) {
  return guarded(ctx, [&] {
    float* part = nullptr;
    B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&part), static_cast<size_t>(colsum_blocks(T)) * N * sizeof(float)));
    try {
      colsum_add(dy, db, part, T, N, ld, ctx->stream);
      ctx->launches += 2;
      B200W_CUDA(cudaStreamSynchronize(ctx->stream));
    } catch (...) { cudaFree(part); throw; }
    cudaFree(part);
  });
}
int b200w_op_rmsnorm_fwd(b200w_ctx* ctx, const void* x, const void* w, void* y, float* rstd, int T,
                         int d, float eps) {
  HOOK(rmsnorm_fwd(x, w, y, rstd, T, d, eps, ctx->stream));
}
int b200w_op_rmsnorm_bwd(b200w_ctx* ctx, const void* dy, const void* x, const void* w,
                         const float* rstd, const void* dresid, void* dx, float* dw, int T, int d) {
  return guarded(ctx, [&] {
    float* part = nullptr;
    B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&part),
                          static_cast<size_t>(rmsnorm_bwd_blocks(T)) * d * sizeof(float)));
    try {
      rmsnorm_bwd(dy, x, w, rstd, dresid, dx, dw, part, T, d, ctx->stream);
      ctx->launches += 2;
      B200W_CUDA(cudaStreamSynchronize(ctx->stream));
    } catch (...) { cudaFree(part); throw; }
    cudaFree(part);
  });
}
int b200w_op_rope(b200w_ctx* ctx, void* buf, int ld, int T, int S, int nheads, int dh, float theta,
                  int inverse) {
  return guarded(ctx, [&] {
    float2* tab = nullptr;
    B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&tab), static_cast<size_t>(S) * (dh / 2) * sizeof(float2)));
    try {
      rope_table(tab, S, dh, theta, ctx->stream);
      rope_apply(buf, ld, tab, T, S, nheads, dh, inverse != 0, ctx->stream);
      ++ctx->launches;
      B200W_CUDA(cudaStreamSynchronize(ctx->stream));
    } catch (...) { cudaFree(tab); throw; }
    cudaFree(tab);
  });
}
int b200w_op_swiglu_fwd(b200w_ctx* ctx, const void* gu, void* h, int T, int f) {
  HOOK(swiglu_fwd(gu, h, T, f, ctx->stream));
}
int b200w_op_swiglu_bwd(b200w_ctx* ctx, const void* dh, const void* gu, void* dgu, int T, int f) {
  HOOK(swiglu_bwd(dh, gu, dgu, T, f, ctx->stream));
}
int b200w_op_ce(b200w_ctx* ctx, void* logits, const int32_t* labels, float* nll, int T, int S, int V,
                float inv_n) {
  return guarded(ctx, [&] {
    int32_t* tg = nullptr;
    B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&tg), static_cast<size_t>(T) * 4));
    try {
      B200W_CUDA(cudaMemcpyAsync(ctx_scal(ctx) + 4, &inv_n, sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
      ce_shift_targets(labels, tg, T, S, ctx->stream);
      ce_loss_fwd_bwd(logits, tg, nll, T, V, ctx_scal(ctx) + 4, ctx->stream);
      ctx->launches += 2;
      B200W_CUDA(cudaStreamSynchronize(ctx->stream));
    } catch (...) { cudaFree(tg); throw; }
    cudaFree(tg);
  });
}
int b200w_op_attention_fwd(b200w_ctx* ctx, const void* qkv, int ld_qkv, int k_off, int v_off,
                           void* out, int ld_out, float* lse2, int B, int S, int H, int Hkv,
                           float scale) {
  HOOK(attention_fwd(qkv, ld_qkv, k_off, v_off, out, ld_out, lse2, B, S, H, Hkv, scale, ctx->stream));
}
int b200w_op_attention_bwd(b200w_ctx* ctx, const void* qkv, int ld_qkv, int k_off, int v_off,
                           const void* out, const void* dout, int ld_out, const float* lse2,
                           float* delta, void* dqkv, int B, int S, int H, int Hkv, float scale) {
  HOOK(attention_bwd(qkv, ld_qkv, k_off, v_off, out, dout, ld_out, lse2, delta, dqkv, B, S, H, Hkv,
                     scale, ctx->stream));
}
}  // extern "C"

namespace {
// runs f(DocBounds) with the bounds of device positions [B * S] derived into scratch (doc_bounds)
template <typename F>
void with_doc_bounds(b200w_ctx* ctx, const int32_t* positions, int B, int S, F&& f) {
  B200W_CHECK(positions, "NULL positions");
  const size_t T = static_cast<size_t>(B) * S;
  int32_t* se = nullptr;
  B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&se), 2 * T * sizeof(int32_t)));
  try {
    doc_bounds(positions, se, se + T, static_cast<int>(T), S, ctx->stream);
    ++ctx->launches;
    const DocBounds db{positions, se, se + T};
    f(db);
    B200W_CUDA(cudaStreamSynchronize(ctx->stream));
  } catch (...) { cudaFree(se); throw; }
  cudaFree(se);
}
}  // namespace

extern "C" {

int b200w_op_attention_fwd_docs(b200w_ctx* ctx, const void* qkv, int ld_qkv, int k_off, int v_off, void* out,
                                int ld_out, float* lse2, const int32_t* positions, int B, int S, int H, int Hkv,
                                float scale) {
  return guarded(ctx, [&] {
    with_doc_bounds(ctx, positions, B, S, [&](const DocBounds& db) {
      attention_fwd(qkv, ld_qkv, k_off, v_off, out, ld_out, lse2, B, S, H, Hkv, scale, ctx->stream, &db);
      ++ctx->launches;
    });
  });
}
int b200w_op_attention_bwd_docs(b200w_ctx* ctx, const void* qkv, int ld_qkv, int k_off, int v_off,
                                const void* out, const void* dout, int ld_out, const float* lse2, float* delta,
                                void* dqkv, const int32_t* positions, int B, int S, int H, int Hkv, float scale) {
  return guarded(ctx, [&] {
    with_doc_bounds(ctx, positions, B, S, [&](const DocBounds& db) {
      attention_bwd(qkv, ld_qkv, k_off, v_off, out, dout, ld_out, lse2, delta, dqkv, B, S, H, Hkv, scale,
                    ctx->stream, &db);
      ctx->launches += 3;
    });
  });
}
int b200w_op_rope_positions(b200w_ctx* ctx, void* buf, int ld, int T, int S, int nheads, int dh, float theta,
                            int inverse, const int32_t* positions) {
  return guarded(ctx, [&] {
    B200W_CHECK(positions, "NULL positions");
    float2* tab = nullptr;
    B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&tab), static_cast<size_t>(S) * (dh / 2) * sizeof(float2)));
    try {
      rope_table(tab, S, dh, theta, ctx->stream);
      rope_apply(buf, ld, tab, T, S, nheads, dh, inverse != 0, ctx->stream, 0, positions);
      ++ctx->launches;
      B200W_CUDA(cudaStreamSynchronize(ctx->stream));
    } catch (...) { cudaFree(tab); throw; }
    cudaFree(tab);
  });
}
int b200w_op_adamw(b200w_ctx* ctx, float* master, float* m, float* v, const void* g, int g_bf16,
                   void* w_bf16, int64_t n, float lr, float beta1, float beta2, float eps, float wd,
                   int step, float gscale) {
  return guarded(ctx, [&] {
    B200W_CUDA(cudaMemcpyAsync(ctx_scal(ctx), &gscale, sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    adamw_step(master, m, v, g, g_bf16 != 0, w_bf16, static_cast<size_t>(n), lr, beta1, beta2, eps, wd, step,
               ctx_scal(ctx), ctx->stream);
    ++ctx->launches;
    B200W_CUDA(cudaStreamSynchronize(ctx->stream));
  });
}
int b200w_op_poison_onchip(b200w_ctx* ctx, uint32_t pattern) {
  return guarded(ctx, [&] {
    static PerDeviceOnce once;
    once.run([&] {
      B200W_CUDA(cudaFuncSetAttribute(poison_onchip_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, POISON_SMEM));
    });
    // one CTA per SM at a time (smem-limited); several waves so that every SM is visited
    poison_onchip_kernel<<<sm_count() * 4, 128, POISON_SMEM, ctx->stream>>>(pattern);
    B200W_CUDA(cudaGetLastError());
    B200W_CUDA(cudaStreamSynchronize(ctx->stream));
  });
}

int b200w_op_grad_norm(b200w_ctx* ctx, const void* g, int g_bf16, int64_t n, float* norm_out) {
  return guarded(ctx, [&] {
    double* ss = nullptr;
    B200W_CUDA(cudaMalloc(reinterpret_cast<void**>(&ss), sizeof(double)));
    B200W_CUDA(cudaMemsetAsync(ss, 0, sizeof(double), ctx->stream));
    grad_sumsq(g, g_bf16 != 0, static_cast<size_t>(n), ss, ctx->stream);
    ++ctx->launches;
    double h = 0;
    B200W_CUDA(cudaMemcpyAsync(&h, ss, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    B200W_CUDA(cudaStreamSynchronize(ctx->stream));
    cudaFree(ss);
    if (norm_out) *norm_out = static_cast<float>(sqrt(h));
  });
}

}  // extern "C"
