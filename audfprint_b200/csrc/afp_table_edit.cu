// HashTable.remove and HashTable.retrieve (reference hash_table.py:346-383) on the device-resident
// table, for a list of ids in one pass over the table.
//
// The requested ids become a bitmap of the id space (one bit per id up to the largest requested
// one; 128 KB covers 2^20 ids) plus an index per id into the request list, read only for entries
// that are in the set.  An entry's id is (value >> maxtimebits) - 1; an empty slot (value 0) gives
// 0xffffffff, outside every set.  Both kernels map one warp to one bucket.
//
// remove: membership and the per-id removed counts are taken over the whole row, as the
// reference's id_in_table does; a bucket holding at least one removed entry keeps its surviving
// entries among slots < min(count, depth), compacted in slot order, the rest of the row is zeroed
// and its count becomes the number of survivors.  Other buckets are not written.  Removing ids
// A and B in one pass leaves the same table as removing A, then B.
//
// retrieve: per bucket, the number of matching entries among slots < min(count, depth); an
// exclusive scan over the buckets gives every bucket its output segment; the entries are written
// as (time, hash) in (hash, slot) order with their request index as key; a stable radix sort by
// that key groups them per requested id without changing that order.
#include <algorithm>
#include <unordered_map>
#include <cub/cub.cuh>
#include "afp_internal.cuh"

namespace {

constexpr int WARPS = 8;   // buckets per 256-thread CTA

__device__ __forceinline__ bool in_set(uint32_t v, int mtb, const uint32_t* bits, uint32_t nbits, uint32_t& id) {
  id = (v >> mtb) - 1u;
  return id < nbits && ((__ldg(&bits[id >> 5]) >> (id & 31u)) & 1u);
}

// bitmap bit + request index of every id; with hpi, the ids' hashesperid is zeroed (remove)
__global__ void afp_edit_idset_kernel(const int64_t* ids, int64_t n, uint32_t* bits, int32_t* slot, uint32_t* hpi) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t id = (uint32_t)ids[k];
  atomicOr(&bits[id >> 5], 1u << (id & 31u));
  slot[id] = (int32_t)k;
  if (hpi) hpi[id] = 0u;
}

__global__ void __launch_bounds__(256) afp_remove_kernel(uint32_t* table, int32_t* counts, int64_t nb, int depth,
                                                         int mtb, const uint32_t* bits, uint32_t nbits,
                                                         const int32_t* slot, unsigned long long* removed) {
  const int64_t b = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5);
  if (b >= nb) return;
  const unsigned lane = threadIdx.x & 31u;
  uint32_t* row = table + (size_t)b * depth;
  bool touched = false;
  for (int s0 = 0; s0 < depth; s0 += 32) {          // membership over the whole row
    const int s = s0 + (int)lane;
    uint32_t id;
    const bool m = s < depth && in_set(row[s], mtb, bits, nbits, id);
    const unsigned mm = __ballot_sync(0xffffffffu, m);
    if (mm == 0u) continue;
    touched = true;
    if (m) {                                          // one atomic per distinct id in these 32 slots
      const unsigned grp = __match_any_sync(mm, id);
      if (lane == (unsigned)(__ffs(grp) - 1)) atomicAdd(&removed[slot[id]], (unsigned long long)__popc(grp));
    }
  }
  if (!touched) return;
  // survivors among the valid slots, in slot order.  Every write lands at or below the slot it
  // came from and the ballot orders this chunk's reads before its writes, so in place is safe.
  const int n = min(counts[b], depth);
  int kept = 0;
  for (int s0 = 0; s0 < n; s0 += 32) {
    const int s = s0 + (int)lane;
    const uint32_t v = s < n ? row[s] : 0u;
    uint32_t id;
    const bool keep = s < n && !in_set(v, mtb, bits, nbits, id);
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    if (keep) row[kept + __popc(km & ((1u << lane) - 1u))] = v;
    kept += __popc(km);
  }
  for (int s = kept + (int)lane; s < depth; s += 32) row[s] = 0u;
  if (lane == 0) counts[b] = kept;
}

__global__ void __launch_bounds__(256) afp_retrieve_count_kernel(const uint32_t* table, const int32_t* counts,
                                                                 int64_t nb, int depth, int mtb, const uint32_t* bits,
                                                                 uint32_t nbits, int32_t* bcnt) {
  const int64_t b = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5);
  if (b >= nb) return;
  const int lane = threadIdx.x & 31;
  const uint32_t* row = table + (size_t)b * depth;
  const int n = min(counts[b], depth);
  int c = 0;
  for (int s0 = 0; s0 < n; s0 += 32) {
    const int s = s0 + lane;
    uint32_t id;
    c += __popc(__ballot_sync(0xffffffffu, s < n && in_set(row[s], mtb, bits, nbits, id)));
  }
  if (lane == 0) bcnt[b] = c;
}

// matching entries of a bucket -> key = request index, value = (time, hash) as one 64-bit word
// (the int32 [2] row in memory), at the bucket's segment in slot order
__global__ void __launch_bounds__(256) afp_retrieve_scatter_kernel(const uint32_t* table, const int32_t* counts,
                                                                   int64_t nb, int depth, int mtb,
                                                                   const uint32_t* bits, uint32_t nbits,
                                                                   const int32_t* slot, const int32_t* bcnt,
                                                                   const int64_t* boff, uint32_t* key,
                                                                   unsigned long long* val, int32_t* ucnt) {
  const int64_t b = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5);
  if (b >= nb || bcnt[b] == 0) return;
  const unsigned lane = threadIdx.x & 31u;
  const uint32_t* row = table + (size_t)b * depth;
  const int n = min(counts[b], depth);
  const uint32_t tmask = (1u << mtb) - 1u;
  int64_t o = boff[b];
  for (int s0 = 0; s0 < n; s0 += 32) {
    const int s = s0 + (int)lane;
    const uint32_t v = s < n ? row[s] : 0u;
    uint32_t id;
    const bool m = s < n && in_set(v, mtb, bits, nbits, id);
    const unsigned mm = __ballot_sync(0xffffffffu, m);
    if (m) {
      const int64_t p = o + __popc(mm & ((1u << lane) - 1u));
      const int32_t u = slot[id];
      key[p] = (uint32_t)u;
      val[p] = (unsigned long long)(v & tmask) | ((unsigned long long)b << 32);
      atomicAdd(&ucnt[u], 1);
    }
    o += __popc(mm);
  }
}

// one CTA per request: the rows of its id (requests may repeat an id)
__global__ void afp_retrieve_gather_kernel(const unsigned long long* val, const int64_t* uoff, const int32_t* req_u,
                                           const int64_t* roff, unsigned long long* out) {
  const int k = blockIdx.x;
  const int u = req_u[k];
  const int64_t s = uoff[u], len = uoff[u + 1] - s, d = roff[k];
  for (int64_t i = threadIdx.x; i < len; i += blockDim.x) out[d + i] = val[s + i];
}

// ids: in [0, nids), each one a table id
int check_ids(afp_ctx* c, const int64_t* ids, int64_t n) {
  for (int64_t k = 0; k < n; ++k)
    if (ids[k] < 0 || ids[k] >= c->tab.nids) AFP_FAIL(c, AFP_ERR_INVALID, "track id outside [0, number of ids)");
  return AFP_OK;
}

// the id set of n distinct ids on the device; *nbits = largest id + 1
int stage_id_set(afp_ctx* c, const int64_t* ids, int64_t n, bool zero_hpi, uint32_t* nbits) {
  const int64_t mx = *std::max_element(ids, ids + n);
  *nbits = (uint32_t)(mx + 1);
  const size_t words = ((size_t)mx + 32) / 32;
  AFP_CUDA(c, c->d_ed_ids.reserve(sizeof(int64_t) * (size_t)n));
  AFP_CUDA(c, c->d_ed_bits.reserve(sizeof(uint32_t) * words));
  AFP_CUDA(c, c->d_ed_slot.reserve(sizeof(int32_t) * ((size_t)mx + 1)));
  AFP_CUDA(c, cudaMemcpyAsync(c->d_ed_ids.p, ids, sizeof(int64_t) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
  AFP_CUDA(c, cudaMemsetAsync(c->d_ed_bits.p, 0, sizeof(uint32_t) * words, c->stream));
  afp_edit_idset_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c->stream>>>(
      c->d_ed_ids.as<int64_t>(), n, c->d_ed_bits.as<uint32_t>(), c->d_ed_slot.as<int32_t>(),
      zero_hpi ? c->tab.hashesperid.as<uint32_t>() : nullptr);
  AFP_CUDA(c, cudaGetLastError());
  c->launches++;
  return AFP_OK;
}

}  // namespace

extern "C" {

int afp_table_remove_ids(afp_ctx* c, const int64_t* ids, int64_t n, int64_t* removed) {
  if (!c || n < 0 || (n > 0 && !ids)) return AFP_ERR_INVALID;
  if (!c->tab.loaded) AFP_FAIL(c, AFP_ERR_STATE, "no table on the device");
  int rc = check_ids(c, ids, n);
  if (rc) return rc;
  std::vector<int64_t> sorted(ids, ids + n);
  std::sort(sorted.begin(), sorted.end());
  if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end())
    AFP_FAIL(c, AFP_ERR_INVALID, "an id is given twice");
  if (n == 0) return AFP_OK;
  AFP_CUDA(c, cudaSetDevice(c->device));
  uint32_t nbits = 0;
  if ((rc = stage_id_set(c, ids, n, true, &nbits))) return rc;
  AFP_CUDA(c, c->d_ed_cnt.reserve(sizeof(unsigned long long) * (size_t)n));
  AFP_CUDA(c, cudaMemsetAsync(c->d_ed_cnt.p, 0, sizeof(unsigned long long) * (size_t)n, c->stream));
  const int64_t nb = (int64_t)1 << c->tab.hashbits;
  afp_remove_kernel<<<(unsigned)((nb + WARPS - 1) / WARPS), 256, 0, c->stream>>>(
      c->tab.table.as<uint32_t>(), c->tab.counts.as<int32_t>(), nb, c->tab.depth, c->tab.maxtimebits,
      c->d_ed_bits.as<uint32_t>(), nbits, c->d_ed_slot.as<int32_t>(), c->d_ed_cnt.as<unsigned long long>());
  AFP_CUDA(c, cudaGetLastError());
  c->launches++;
  if (removed)
    AFP_CUDA(c, cudaMemcpyAsync(removed, c->d_ed_cnt.p, sizeof(int64_t) * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  // hashesperid lost zeros-to-be and the table lost entries: the matcher's pruning bound and its
  // check for live entries of zero-length tracks are recomputed
  return afp_table_stats(c);
}

int afp_table_retrieve_ids(afp_ctx* c, const int64_t* ids, int64_t n, int64_t* total_rows) {
  if (!c || n < 0 || (n > 0 && !ids)) return AFP_ERR_INVALID;
  if (!c->tab.loaded) AFP_FAIL(c, AFP_ERR_STATE, "no table on the device");
  c->rt_total = -1;
  int rc = check_ids(c, ids, n);
  if (rc) return rc;
  if (n >= ((int64_t)1 << 31)) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "more than 2^31 ids in one call");
  // distinct ids in first-request order; every request points at its id's slot
  std::unordered_map<int64_t, int32_t> first;
  std::vector<int64_t> uids;
  std::vector<int32_t> req_u((size_t)n);
  for (int64_t k = 0; k < n; ++k) {
    auto it = first.emplace(ids[k], (int32_t)uids.size());
    if (it.second) uids.push_back(ids[k]);
    req_u[(size_t)k] = it.first->second;
  }
  const int64_t nu = (int64_t)uids.size();
  c->h_rt_off.assign((size_t)n + 1, 0);
  if (n == 0) {
    c->rt_total = 0;
    if (total_rows) *total_rows = 0;
    return AFP_OK;
  }
  AFP_CUDA(c, cudaSetDevice(c->device));
  uint32_t nbits = 0;
  if ((rc = stage_id_set(c, uids.data(), nu, false, &nbits))) return rc;
  const int64_t nb = (int64_t)1 << c->tab.hashbits;
  const int mtb = c->tab.maxtimebits, depth = c->tab.depth;
  AFP_CUDA(c, c->d_ed_cnt.reserve(sizeof(int32_t) * (size_t)nb));
  AFP_CUDA(c, c->d_ed_off.reserve(sizeof(int64_t) * (size_t)(nb + 1)));
  AFP_CUDA(c, c->d_ed_uoff.reserve(sizeof(int32_t) * (size_t)nu + sizeof(int64_t) * (size_t)(nu + 1)));
  int32_t* bcnt = c->d_ed_cnt.as<int32_t>();
  int64_t* boff = c->d_ed_off.as<int64_t>();
  int64_t* uoff = c->d_ed_uoff.as<int64_t>();
  int32_t* ucnt = reinterpret_cast<int32_t*>(uoff + nu + 1);
  const unsigned grid = (unsigned)((nb + WARPS - 1) / WARPS);
  afp_retrieve_count_kernel<<<grid, 256, 0, c->stream>>>(c->tab.table.as<uint32_t>(), c->tab.counts.as<int32_t>(), nb,
                                                         depth, mtb, c->d_ed_bits.as<uint32_t>(), nbits, bcnt);
  AFP_CUDA(c, cudaGetLastError());
  c->launches++;
  if ((rc = afp_scan_large(c, bcnt, boff, nb))) return rc;
  int64_t M = 0;
  AFP_CUDA(c, cudaMemcpyAsync(&M, boff + nb, sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
  AFP_CUDA(c, cudaMemsetAsync(ucnt, 0, sizeof(int32_t) * (size_t)nu, c->stream));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  if (M >= ((int64_t)1 << 31)) AFP_FAIL(c, AFP_ERR_UNSUPPORTED, "more than 2^31 rows in one retrieve");
  c->rt_src = 0;
  if (M > 0) {
    AFP_CUDA(c, c->d_ed_key.reserve(sizeof(uint32_t) * (size_t)M));
    AFP_CUDA(c, c->d_ed_val.reserve(sizeof(unsigned long long) * (size_t)M));
    afp_retrieve_scatter_kernel<<<grid, 256, 0, c->stream>>>(
        c->tab.table.as<uint32_t>(), c->tab.counts.as<int32_t>(), nb, depth, mtb, c->d_ed_bits.as<uint32_t>(), nbits,
        c->d_ed_slot.as<int32_t>(), bcnt, boff, c->d_ed_key.as<uint32_t>(), c->d_ed_val.as<unsigned long long>(), ucnt);
    AFP_CUDA(c, cudaGetLastError());
    c->launches++;
    if (nu > 1) {      // stable: within one id the (hash, slot) order of the scatter is kept
      int end_bit = 1;
      while (((int64_t)1 << end_bit) < nu) ++end_bit;
      size_t tmp = 0;
      AFP_CUDA(c, c->d_ed_key2.reserve(sizeof(uint32_t) * (size_t)M));
      AFP_CUDA(c, c->d_ed_val2.reserve(sizeof(unsigned long long) * (size_t)M));
      AFP_CUDA(c, cub::DeviceRadixSort::SortPairs(nullptr, tmp, c->d_ed_key.as<uint32_t>(), c->d_ed_key2.as<uint32_t>(),
                                                  c->d_ed_val.as<unsigned long long>(),
                                                  c->d_ed_val2.as<unsigned long long>(), (int)M, 0, end_bit, c->stream));
      AFP_CUDA(c, c->d_ed_cub.reserve(tmp));
      AFP_CUDA(c, cub::DeviceRadixSort::SortPairs(c->d_ed_cub.p, tmp, c->d_ed_key.as<uint32_t>(),
                                                  c->d_ed_key2.as<uint32_t>(), c->d_ed_val.as<unsigned long long>(),
                                                  c->d_ed_val2.as<unsigned long long>(), (int)M, 0, end_bit, c->stream));
      c->launches++;
      c->rt_src = 1;
    }
  }
  if ((rc = afp_launch_scan_i32_to_i64(c, ucnt, uoff, nu))) return rc;
  std::vector<int64_t> h_uoff((size_t)nu + 1);
  AFP_CUDA(c, cudaMemcpyAsync(h_uoff.data(), uoff, sizeof(int64_t) * (size_t)(nu + 1), cudaMemcpyDeviceToHost, c->stream));
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  for (int64_t k = 0; k < n; ++k) {
    const int32_t u = req_u[(size_t)k];
    c->h_rt_off[(size_t)k + 1] = c->h_rt_off[(size_t)k] + h_uoff[(size_t)u + 1] - h_uoff[(size_t)u];
  }
  const int64_t total = c->h_rt_off[(size_t)n];
  if (nu < n && total > 0) {       // a repeated id: copy its rows once per request
    const unsigned long long* src = c->rt_src ? c->d_ed_val2.as<unsigned long long>() : c->d_ed_val.as<unsigned long long>();
    AFP_CUDA(c, c->d_ed_req.reserve(sizeof(int64_t) * (size_t)(n + 1) + sizeof(int32_t) * (size_t)n));
    AFP_CUDA(c, c->d_ed_rows.reserve(sizeof(unsigned long long) * (size_t)total));
    int64_t* d_roff = c->d_ed_req.as<int64_t>();
    int32_t* d_requ = reinterpret_cast<int32_t*>(d_roff + n + 1);
    AFP_CUDA(c, cudaMemcpyAsync(d_roff, c->h_rt_off.data(), sizeof(int64_t) * (size_t)(n + 1), cudaMemcpyHostToDevice,
                                c->stream));
    AFP_CUDA(c, cudaMemcpyAsync(d_requ, req_u.data(), sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    afp_retrieve_gather_kernel<<<(unsigned)n, 128, 0, c->stream>>>(src, uoff, d_requ, d_roff,
                                                                  c->d_ed_rows.as<unsigned long long>());
    AFP_CUDA(c, cudaGetLastError());
    c->launches++;
    AFP_CUDA(c, cudaStreamSynchronize(c->stream));      // req_u and h_rt_off are host memory being read
    c->rt_src = 2;
  }
  c->rt_total = total;
  if (total_rows) *total_rows = total;
  return AFP_OK;
}

int afp_fetch_retrieved(afp_ctx* c, int32_t* rows, int rows_on_host, int64_t* row_offsets) {
  if (!c) return AFP_ERR_INVALID;
  if (c->rt_total < 0) AFP_FAIL(c, AFP_ERR_STATE, "afp_table_retrieve_ids has not been called");
  AFP_CUDA(c, cudaSetDevice(c->device));
  if (row_offsets) std::copy(c->h_rt_off.begin(), c->h_rt_off.end(), row_offsets);
  if (rows && c->rt_total > 0) {
    const DevBuf& src = c->rt_src == 2 ? c->d_ed_rows : (c->rt_src == 1 ? c->d_ed_val2 : c->d_ed_val);
    AFP_CUDA(c, cudaMemcpyAsync(rows, src.p, sizeof(int32_t) * 2 * (size_t)c->rt_total,
                                rows_on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, c->stream));
  }
  AFP_CUDA(c, cudaStreamSynchronize(c->stream));
  return AFP_OK;
}

}  // extern "C"
