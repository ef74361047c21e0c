// eqf_abi.cu - plan construction, error reporting and misc entry points of libeqf_b200.so.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "eqf_common.cuh"

namespace eqf {

static thread_local std::string g_last_error;

void set_error(const std::string& msg) { g_last_error = msg; }

int check_cuda(cudaError_t err, const char* what) {
  if (err == cudaSuccess) return EQF_OK;
  g_last_error = std::string(what) + ": " + cudaGetErrorString(err);
  return EQF_ERR_CUDA;
}

static std::mutex g_upload_mutex;

static std::vector<const GeneratedKernels*>& generated_registry() {
  static std::vector<const GeneratedKernels*> reg;
  return reg;
}
int register_generated(const GeneratedKernels* k) { generated_registry().push_back(k); return (int)generated_registry().size(); }
const GeneratedKernels* find_generated(unsigned long long signature) {
  for (const GeneratedKernels* k : generated_registry()) if (k->signature == signature) return k;
  return nullptr;
}

static unsigned long long fnv1a(unsigned long long h, const void* data, size_t n) {
  const unsigned char* p = static_cast<const unsigned char*>(data);
  for (size_t i = 0; i < n; ++i) { h ^= p[i]; h *= 0x100000001B3ULL; }
  return h;
}

// Upload the table blob on first use (plan creation itself needs no GPU).
int ensure_device(const EqfPlan* cplan) {
  EqfPlan* plan = const_cast<EqfPlan*>(cplan);
  int dev = 0;
  int rc = check_cuda(cudaGetDevice(&dev), "cudaGetDevice");
  if (rc != EQF_OK) return rc;
  std::lock_guard<std::mutex> lock(g_upload_mutex);
  if (plan->d_blob != nullptr && plan->device == dev) return EQF_OK;
  if (plan->d_blob != nullptr) { cudaFree(plan->d_blob); plan->d_blob = nullptr; }
  rc = check_cuda(cudaMalloc(&plan->d_blob, plan->blob.size() * sizeof(uint32_t)), "cudaMalloc(plan blob)");
  if (rc != EQF_OK) return rc;
  rc = check_cuda(cudaMemcpy(plan->d_blob, plan->blob.data(), plan->blob.size() * sizeof(uint32_t),
                             cudaMemcpyHostToDevice), "cudaMemcpy(plan blob)");
  if (rc != EQF_OK) return rc;
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && sms > 0) plan->sm_count = sms;
  plan->device = dev;
  return EQF_OK;
}

}  // namespace eqf

using namespace eqf;

extern "C" int eqf_version(void) { return 100; }

extern "C" const char* eqf_last_error(void) { return g_last_error.c_str(); }

extern "C" int eqf_device_sm_count(void) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return EQF_ERR_CUDA;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return EQF_ERR_CUDA;
  return sms;
}

extern "C" int eqf_plan_create(const EqfPathDesc* paths, int32_t n_paths, const int32_t* in1_l, const int32_t* in1_mul,
                               int32_t n_in1, const int32_t* out_l, const int32_t* out_mul, int32_t n_out, int32_t d_y,
                               int32_t weight_numel, const float* cg, int32_t cg_len, EqfPlan** plan_out) {
  if (plan_out == nullptr) { set_error("plan_out is null"); return EQF_ERR_INVALID; }
  *plan_out = nullptr;
  if (paths == nullptr || in1_l == nullptr || in1_mul == nullptr || out_l == nullptr || out_mul == nullptr || cg == nullptr) {
    set_error("eqf_plan_create: null argument"); return EQF_ERR_INVALID;
  }
  if (n_paths < 1 || n_paths > 4096) { set_error("n_paths out of range"); return EQF_ERR_INVALID; }
  if (n_in1 < 1 || n_in1 > EQF_MAX_BLOCKS || n_out < 1 || n_out > EQF_MAX_BLOCKS) {
    set_error("too many irrep blocks (EQF_MAX_BLOCKS)"); return EQF_ERR_UNSUPPORTED;
  }
  if (d_y < 1 || weight_numel < 1 || cg_len < 1) { set_error("bad sizes"); return EQF_ERR_INVALID; }

  EqfPlan* plan = new EqfPlan();
  PlanHdr& h = plan->hdr;
  std::memset(&h, 0, sizeof(h));
  h.n_paths = n_paths; h.n_in1 = n_in1; h.n_out = n_out; h.d_y = d_y; h.w_numel = weight_numel; h.cg_len = cg_len;
  for (int b = 0; b < n_in1; ++b) {
    if (in1_l[b] < 0 || 2 * in1_l[b] + 1 > kMaxDtpD || in1_mul[b] < 1) {
      delete plan; set_error("in1 degree must be 0.." + std::to_string(EQF_MAX_DEGREE) + " and mul >= 1");
      return EQF_ERR_UNSUPPORTED;
    }
    h.in1_d[b] = 2 * in1_l[b] + 1; h.in1_mul[b] = in1_mul[b];
  }
  for (int g = 0; g < n_out; ++g) {
    if (out_l[g] < 0 || 2 * out_l[g] + 1 > kMaxDtpD || out_mul[g] < 1) {
      delete plan; set_error("output degree must be 0.." + std::to_string(EQF_MAX_DEGREE) + " and mul >= 1");
      return EQF_ERR_UNSUPPORTED;
    }
    h.out_d[g] = 2 * out_l[g] + 1; h.out_mul[g] = out_mul[g];
  }

  std::vector<PathDev> pd(n_paths);
  int m_size = 0;
  for (int p = 0; p < n_paths; ++p) {
    const EqfPathDesc& s = paths[p];
    PathDev& d = pd[p];
    const bool tri = s.l3 >= std::abs(s.l1 - s.l2) && s.l3 <= s.l1 + s.l2;
    // d1, d3 <= kMaxDtpD: the table-walk kernels dispatch on them at compile time (EQF_DISPATCH_D); up to 9 they also fit
    // mdesc's 4-bit fields
    if (s.l1 < 0 || s.l2 < 0 || s.l3 < 0 || !tri || 2 * s.l1 + 1 > kMaxDtpD || 2 * s.l3 + 1 > kMaxDtpD || 2 * s.l2 + 1 > 15) {
      delete plan; set_error("path degrees unsupported or violate the triangle rule"); return EQF_ERR_UNSUPPORTED;
    }
    d.d1 = 2 * s.l1 + 1; d.d2 = 2 * s.l2 + 1; d.d3 = 2 * s.l3 + 1;
    if (s.in1_block < 0 || s.in1_block >= n_in1 || s.out_group < 0 || s.out_group >= n_out) {
      delete plan; set_error("path references a missing block"); return EQF_ERR_INVALID;
    }
    if (h.in1_d[s.in1_block] != d.d1 || h.in1_mul[s.in1_block] != s.mul || h.out_d[s.out_group] != d.d3) {
      delete plan; set_error("path is inconsistent with its in1 block / output group"); return EQF_ERR_INVALID;
    }
    if (s.in2_off < 0 || s.in2_off + d.d2 > d_y || s.w_off < 0 || s.w_off + s.mul > weight_numel ||
        s.out_chan_off < 0 || s.out_chan_off + s.mul > h.out_mul[s.out_group] || s.cg_off < 0 ||
        s.cg_off + d.d1 * d.d2 * d.d3 > cg_len) {
      delete plan; set_error("path offsets out of range"); return EQF_ERR_INVALID;
    }
    d.mul = s.mul; d.xb = s.in1_block; d.y_off = s.in2_off; d.og = s.out_group; d.koff = s.out_chan_off;
    d.w_off = s.w_off; d.cg_off = s.cg_off; d.m_off = m_size; d.pad = 0;
    m_size += d.d1 * d.d3;
  }
  h.m_size = m_size;

  // task tables
  std::vector<int> wtasks, xtasks, xbstart, xbpaths, mdesc(m_size);
  for (int p = 0; p < n_paths; ++p) {
    for (int u0 = 0; u0 < pd[p].mul; u0 += 32) { wtasks.push_back(p); wtasks.push_back(u0); }
    for (int i = 0; i < pd[p].d1; ++i)
      for (int k = 0; k < pd[p].d3; ++k) mdesc[pd[p].m_off + i * pd[p].d3 + k] = (p << 8) | (i << 4) | k;
  }
  for (int b = 0; b < n_in1; ++b) {
    for (int u0 = 0; u0 < h.in1_mul[b]; u0 += 32) { xtasks.push_back(b); xtasks.push_back(u0); }
    xbstart.push_back((int)xbpaths.size());
    for (int p = 0; p < n_paths; ++p) if (pd[p].xb == b) xbpaths.push_back(p);
  }
  xbstart.push_back((int)xbpaths.size());
  h.n_wtasks = (int)wtasks.size() / 2;
  h.n_xtasks = (int)xtasks.size() / 2;

  // tile size: largest of {8,4,2,1} edges whose scratch fits comfortably beside the tables
  int te = 8;
  const size_t fixed_words = (size_t)n_paths * (sizeof(PathDev) / 4) + cg_len + m_size + 4 * (size_t)n_paths + 64;
  auto scalar_smem = [&](int t) {
    size_t extra = (size_t)std::max(weight_numel, t * m_size);
    return sizeof(uint32_t) * (fixed_words + (size_t)t * m_size + (size_t)t * d_y + extra);
  };
  while (te > 1 && scalar_smem(te) > 40 * 1024) te >>= 1;
  h.te = te;

  h.d_in = 0;
  for (int b = 0; b < n_in1; ++b) { h.in1_off[b] = h.d_in; h.d_in += h.in1_d[b] * h.in1_mul[b]; }

  // vector (float4-per-lane) task tables for one tile of `te` edges
  bool vec_ok = true;
  for (int b = 0; b < n_in1; ++b) vec_ok = vec_ok && (h.in1_mul[b] % 4 == 0);
  for (int g = 0; g < n_out; ++g) vec_ok = vec_ok && (h.out_mul[g] % 4 == 0);
  for (int p = 0; p < n_paths; ++p) vec_ok = vec_ok && (pd[p].koff % 4 == 0) && (pd[p].w_off % 4 == 0);
  vec_ok = vec_ok && (weight_numel % 4 == 0);
  h.vec_ok = vec_ok ? 1 : 0;
  std::vector<int> vwtasks, vxtasks;
  if (vec_ok) {
    for (int b = 0; b < n_in1; ++b) {
      const int nvec = h.in1_mul[b] / 4;
      h.in1_lpe[b] = nvec < 32 ? nvec : 32;
      h.in1_epw[b] = 32 / h.in1_lpe[b];
      h.in1_lpe_shift[b] = -1;
      for (int sft = 0; sft <= 5; ++sft) if ((1 << sft) == h.in1_lpe[b]) h.in1_lpe_shift[b] = sft;
    }
    auto emit = [&](std::vector<int>& out, int id, int b) {
      const int nvec = h.in1_mul[b] / 4;
      const int chunks = (nvec + 31) / 32;
      const int epw = h.in1_epw[b];
      for (int e_start = 0; e_start < te; e_start += epw)
        for (int c = 0; c < chunks; ++c) { out.push_back(id); out.push_back((e_start << 16) | c); }
    };
    for (int p = 0; p < n_paths; ++p) emit(vwtasks, p, pd[p].xb);
    for (int b = 0; b < n_in1; ++b) emit(vxtasks, b, b);
  }
  h.n_vwtasks = (int)vwtasks.size() / 2;
  h.n_vxtasks = (int)vxtasks.size() / 2;

  std::vector<uint32_t>& blob = plan->blob;
  auto align2 = [&]() { if (blob.size() & 1) blob.push_back(0); };
  auto append_ints = [&](const std::vector<int>& v) {
    int off = (int)blob.size();
    for (int x : v) blob.push_back((uint32_t)x);
    return off;
  };
  align2();
  h.off_paths = (int)blob.size();
  blob.resize(blob.size() + (size_t)n_paths * (sizeof(PathDev) / 4));
  std::memcpy(blob.data() + h.off_paths, pd.data(), (size_t)n_paths * sizeof(PathDev));
  h.off_cg = (int)blob.size();
  blob.resize(blob.size() + cg_len);
  std::memcpy(blob.data() + h.off_cg, cg, (size_t)cg_len * sizeof(float));
  h.off_mdesc = append_ints(mdesc);
  align2(); h.off_wtasks = append_ints(wtasks);
  align2(); h.off_xtasks = append_ints(xtasks);
  h.off_xbstart = append_ints(xbstart);
  h.off_xbpaths = append_ints(xbpaths);
  align2(); h.off_vwtasks = append_ints(vwtasks);
  align2(); h.off_vxtasks = append_ints(vxtasks);
  while (blob.size() & 3) blob.push_back(0);   // keep the float scratch behind it 16-byte aligned
  h.blob_words = (int)blob.size();

  auto al4 = [](size_t v) { return (v + 3) & ~(size_t)3; };
  auto smem_for = [&](int t) {
    size_t extra = (size_t)std::max(weight_numel, t * m_size);
    return sizeof(uint32_t) * ((size_t)h.blob_words + (size_t)t * m_size + (size_t)t * d_y + extra);
  };
  if (smem_for(te) > 200 * 1024) { delete plan; set_error("plan tables exceed shared memory"); return EQF_ERR_UNSUPPORTED; }
  plan->smem_bytes = smem_for(te);
  const size_t vec_base = (size_t)h.blob_words + al4((size_t)te * m_size) + al4((size_t)te * d_y) + al4(weight_numel);
  plan->smem_bytes_vec_bwd = sizeof(uint32_t) * vec_base + 16;
  plan->smem_bytes_vec_fwd = sizeof(uint32_t) * (vec_base + 2 * (size_t)te * weight_numel) + 32;
  if (plan->smem_bytes_vec_fwd > 220 * 1024) h.vec_ok = 0;  // weight ring does not fit: scalar kernels
  {  // canonical image hashed exactly like codegen.plan_signature
    std::vector<int32_t> words;
    words.push_back(n_in1);
    for (int b = 0; b < n_in1; ++b) { words.push_back(in1_l[b]); words.push_back(in1_mul[b]); }
    words.push_back(n_out);
    for (int g = 0; g < n_out; ++g) { words.push_back(out_l[g]); words.push_back(out_mul[g]); }
    words.push_back(d_y); words.push_back(weight_numel); words.push_back(n_paths);
    for (int p = 0; p < n_paths; ++p) {
      const EqfPathDesc& s = paths[p];
      const int32_t v[10] = {s.l1, s.l2, s.l3, s.mul, s.in1_block, s.in2_off, s.out_group, s.out_chan_off, s.w_off, s.cg_off};
      words.insert(words.end(), v, v + 10);
    }
    unsigned long long hsh = fnv1a(0xCBF29CE484222325ULL, words.data(), words.size() * sizeof(int32_t));
    hsh = fnv1a(hsh, cg, (size_t)cg_len * sizeof(float));
    plan->signature = hsh;
    plan->gen = find_generated(hsh);
  }
  *plan_out = plan;
  return EQF_OK;
}

extern "C" void eqf_plan_destroy(EqfPlan* plan) {
  if (plan == nullptr) return;
  if (plan->d_blob != nullptr) cudaFree(plan->d_blob);
  delete plan;
}

extern "C" int eqf_plan_info(const EqfPlan* plan, int32_t* out, int32_t n) {
  if (plan == nullptr || out == nullptr) { set_error("eqf_plan_info: null argument"); return EQF_ERR_INVALID; }
  const PlanHdr& h = plan->hdr;
  const int32_t vals[13] = {h.n_paths, h.m_size, h.n_wtasks, h.n_xtasks, h.te, (int32_t)plan->smem_bytes, h.blob_words,
                            h.w_numel, h.vec_ok, h.n_vwtasks, h.n_vxtasks, (int32_t)plan->smem_bytes_vec_fwd,
                            plan->gen != nullptr ? 1 : 0};
  for (int i = 0; i < n && i < 13; ++i) out[i] = vals[i];
  return EQF_OK;
}
