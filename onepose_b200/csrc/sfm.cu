// An object's SfM post-processing on the GPU: the steps of the reference's run.py postprocess (:142-163) between COLMAP's
// model and the 3D annotation files, once the model is read and the images' features extracted.
//   filter_tkl.get_tkl        :35-52    the track-length threshold                                  opb_sfm_filter_points
//   filter_points.filter_3d   :8-83     track length >= threshold, inside the 3D box, by id        opb_sfm_filter_points
//   filter_points.merge       :86-117   close points merged greedily, np.mean of each group        opb_sfm_merge_points
//   feature_process.get_kpt_ann         each group's observations, group-major (:95-188, :320-363)  opb_sfm_gather_observations
//                                       and their descriptors and scores in that order               opb_sfm_gather_features
//   feature_process.count_features      each image's 2D-3D pairs, one per group (:95-135, :197-230) opb_sfm_assign_pairs
//                   + get_assign_matrix
// Every count (kept points, groups, observations) stays on the device: a later step reads it from the scalar an earlier one
// wrote, and launches for the capacity the caller sized.  The arithmetic is the reference's, one rounding per operation
// (__fadd_rn and friends, no fused multiply-add); the model is tests/sfm_reference.py and DESIGN §5.13 states the rules.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <cub/block/block_radix_sort.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>

#include "../../include/onepose_b200.h"
#include "block.cuh"
#include "host_util.cuh"

namespace opb {
namespace {

constexpr int kFilterThreads = 1024;
constexpr int kWarpsPerBlock = 8;
constexpr int32_t kNoSlot = INT32_MAX;

__host__ __device__ inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// ---- the track-length threshold and the box test ----

// filter_by_3d_box's c0 < m && m < v.v on one axis: m = (p - c4) . v in fp32, the three products summed left to right.
__device__ __forceinline__ float dot3(const float* a, const float* b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a[0], b[0]), __fmul_rn(a[1], b[1])), __fmul_rn(a[2], b[2]));
}

// One block walks the points in ascending id order.  get_tkl's threshold is the smallest length L present with at most
// max_num_kp3d points longer than L: the sorted lengths' entry max(P - 1 - max_num_kp3d, 0).  A point is kept when its length
// is at least that and it lies strictly inside the box; a block scan gives each kept point its slot.
__global__ void __launch_bounds__(kFilterThreads) filter_kernel(const double* __restrict__ xyz, const int64_t* __restrict__ track_len,
                                                                const int64_t* __restrict__ ids, int P, const int64_t* __restrict__ sorted_len,
                                                                int k0, const double* __restrict__ corners, int64_t* __restrict__ kept_ids,
                                                                float* __restrict__ kept_xyz, int64_t* __restrict__ track_length,
                                                                int64_t* __restrict__ n_kept) {
  __shared__ int sh[kFilterThreads / 32];
  const int64_t tl = sorted_len[k0];
  float c4[3], v[3][3], vv[3];
  const int axis_corner[3] = {5, 0, 7};                       // v45, v40, v47
  for (int a = 0; a < 3; ++a) c4[a] = __double2float_rn(corners[4 * 3 + a]);
  for (int k = 0; k < 3; ++k) {
    for (int a = 0; a < 3; ++a) v[k][a] = __fsub_rn(__double2float_rn(corners[axis_corner[k] * 3 + a]), c4[a]);
    vv[k] = dot3(v[k], v[k]);
  }
  int base = 0;
  for (int start = 0; start < P; start += kFilterThreads) {
    const int i = start + (int)threadIdx.x;
    bool kept = false;
    float p[3];
    if (i < P && track_len[i] >= tl) {
      float d[3];
      for (int a = 0; a < 3; ++a) {
        p[a] = __double2float_rn(xyz[(size_t)i * 3 + a]);
        d[a] = __fsub_rn(p[a], c4[a]);
      }
      kept = true;
      for (int k = 0; k < 3; ++k) {
        const float m = dot3(d, v[k]);
        kept = kept && 0.0f < m && m < vv[k];
      }
    }
    int total;
    const int slot = base + block_rank(kept, sh, &total);
    if (kept) {
      kept_ids[slot] = ids[i];
      for (int a = 0; a < 3; ++a) kept_xyz[(size_t)slot * 3 + a] = p[a];
    }
    base += total;
  }
  if (threadIdx.x == 0) {
    *track_length = tl;
    *n_kept = base;
  }
}

// ---- the merge ----

// scipy's pdist 'euclidean' of two fp32 rows widened to fp64: s = dx*dx, s += dy*dy, s += dz*dz, a correctly rounded sqrt.
__device__ __forceinline__ double pdist(const float* a, const float* b) {
  double s = 0.0;
  for (int k = 0; k < 3; ++k) {
    const double d = __dsub_rn((double)a[k], (double)b[k]);
    s = k == 0 ? __dmul_rn(d, d) : __dadd_rn(s, __dmul_rn(d, d));
  }
  return __dsqrt_rn(s);
}

// One warp per row j < n: the number of points closer than the threshold, j itself included (a ballot and popc per 32 points).
__global__ void neighbour_count_kernel(const float* __restrict__ xyz, const int64_t* __restrict__ n_dev, int cap, double threshold,
                                       int32_t* __restrict__ count) {
  const int n = (int)*n_dev;
  const int lane = threadIdx.x & 31;
  const int j = (int)(blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5));
  if (j >= n || j >= cap) return;
  const float pj[3] = {xyz[(size_t)j * 3], xyz[(size_t)j * 3 + 1], xyz[(size_t)j * 3 + 2]};
  int c = 0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    const bool near = i < n && pdist(pj, xyz + (size_t)i * 3) < threshold;
    c += __popc(__ballot_sync(0xffffffffu, near));
  }
  if (lane == 0) count[j] = c;
}

// merge's greedy pass in one warp, j = 0 .. n - 1 in order.  A point whose list is itself alone is a group unless recorded.  A
// longer list is walked 32 points at a time, its members written in ascending index order behind the groups so far; the walk
// stops at the first chunk that holds a recorded member, before writing it (j is skipped), otherwise the list becomes a group
// and its members are recorded.  Only unrecorded points are ever written, so no write reaches past row n - 1.
// The group's position is np.mean of its fp32 rows: an fp32 sum from +0.0 in member order, then an fp32 divide by the count.
__global__ void __launch_bounds__(32) merge_greedy_kernel(const float* __restrict__ xyz, const int64_t* __restrict__ ids,
                                                           const int64_t* __restrict__ n_dev, int cap, double threshold,
                                                           const int32_t* __restrict__ count, int32_t* __restrict__ recorded,
                                                           double* __restrict__ merged, int32_t* __restrict__ offsets,
                                                           int32_t* __restrict__ member_src, int64_t* __restrict__ member_ids,
                                                           int32_t* __restrict__ slot_of, int64_t* __restrict__ n_groups,
                                                           int64_t* __restrict__ n_members) {
  const int n = min((int)*n_dev, cap);
  const int lane = threadIdx.x;
  for (int i = lane; i < n; i += 32) {
    recorded[i] = 0;
    slot_of[i] = kNoSlot;
  }
  __syncwarp();
  int groups = 0, cursor = 0;
  if (lane == 0) offsets[0] = 0;
  for (int j = 0; j < n; ++j) {
    int len = 0;
    if (count[j] == 1) {
      if (recorded[j]) continue;
      if (lane == 0) member_src[cursor] = j;
      len = 1;
    } else {
      const float pj[3] = {xyz[(size_t)j * 3], xyz[(size_t)j * 3 + 1], xyz[(size_t)j * 3 + 2]};
      bool taken = false;
      for (int i0 = 0; i0 < n && !taken; i0 += 32) {
        const int i = i0 + lane;
        const bool near = i < n && pdist(pj, xyz + (size_t)i * 3) < threshold;
        const unsigned m = __ballot_sync(0xffffffffu, near);
        taken = __ballot_sync(0xffffffffu, near && recorded[i]) != 0;
        if (taken) break;
        // every point written so far is unrecorded and distinct, so cursor + len stays below n
        if (near) member_src[cursor + len + __popc(m & ((1u << lane) - 1u))] = i;
        len += __popc(m);
      }
      if (taken) continue;
    }
    __syncwarp();
    for (int k = lane; k < len; k += 32) {
      const int i = member_src[cursor + k];
      recorded[i] = 1;
      slot_of[i] = cursor + k;
      member_ids[cursor + k] = ids[i];
    }
    if (lane == 0) {
      float s[3] = {0.0f, 0.0f, 0.0f};
      for (int k = 0; k < len; ++k)
        for (int a = 0; a < 3; ++a) s[a] = __fadd_rn(s[a], xyz[(size_t)member_src[cursor + k] * 3 + a]);
      for (int a = 0; a < 3; ++a) merged[(size_t)groups * 3 + a] = (double)__fdiv_rn(s[a], (float)len);
      offsets[groups + 1] = cursor + len;
    }
    __syncwarp();
    cursor += len;
    ++groups;
  }
  if (lane == 0) {
    *n_groups = groups;
    *n_members = cursor;
  }
}

// ---- the observations ----

// One thread per feature (f, k), k < counts[f]: its point's slot in the merge's member order, found by binary search of the id
// among the kept ids (ascending), or kNoSlot.  The value is the feature's flat index f * cap + k.  Per-slot counts are added.
__global__ void observation_keys_kernel(const int64_t* __restrict__ point3d_ids, const int32_t* __restrict__ counts, int F, int cap,
                                        const int64_t* __restrict__ kept_ids, const int64_t* __restrict__ n_kept_dev, int kept_cap,
                                        const int32_t* __restrict__ slot_of, int32_t* __restrict__ keys, int32_t* __restrict__ vals,
                                        int32_t* __restrict__ slot_count) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)F * cap) return;
  const int f = (int)(t / cap), k = (int)(t % cap);
  int32_t key = kNoSlot;
  if (k < counts[f]) {
    const int64_t id = point3d_ids[t];
    int lo = 0, hi = min((int)*n_kept_dev, kept_cap);
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (kept_ids[mid] < id) lo = mid + 1;
      else hi = mid;
    }
    if (id != -1 && lo < min((int)*n_kept_dev, kept_cap) && kept_ids[lo] == id) key = slot_of[lo];
  }
  keys[t] = key;
  vals[t] = (int32_t)t;
  if (key != kNoSlot) atomicAdd(slot_count + key, 1);
}

// One thread per group: its observation count (idxs) is the sum over its members; the total is added up, and the first member
// without an observation (the reference's KeyError) is kept as the smallest such slot.
__global__ void group_counts_kernel(const int32_t* __restrict__ offsets, const int64_t* __restrict__ n_groups_dev, int cap,
                                    const int32_t* __restrict__ slot_count, int64_t* __restrict__ idxs, unsigned long long* __restrict__ total,
                                    int64_t* __restrict__ missing) {
  const int g = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (g >= min((int)*n_groups_dev, cap)) return;
  int64_t s = 0;
  for (int m = offsets[g]; m < offsets[g + 1]; ++m) {
    s += slot_count[m];
    if (slot_count[m] == 0) atomicMin((unsigned long long*)missing, (unsigned long long)m);
  }
  idxs[g] = s;
  atomicAdd(total, (unsigned long long)s);
}

// Row r of the collected observations: the descriptor column and score of feature order[r], widened to fp64.
__global__ void gather_features_kernel(const int32_t* __restrict__ order, int64_t total, int cap, int D, const float* __restrict__ scores,
                                       const float* __restrict__ desc, double* __restrict__ out_desc, double* __restrict__ out_scores) {
  const int64_t r = blockIdx.x;
  if (r >= total) return;
  const int t = order[r];
  const int f = t / cap, k = t % cap;
  const float* src = desc + (size_t)f * D * cap + k;
  for (int d = threadIdx.x; d < D; d += blockDim.x) out_desc[(size_t)r * D + d] = (double)src[(size_t)d * cap];
  if (threadIdx.x == 0) out_scores[r] = (double)scores[t];
}

// ---- the 2D-3D pairs of each image ----

// count_features keeps, per image, {kept id: its last feature index} in the order of each id's first feature; get_assign_matrix
// walks that and pairs an id with its group unless the group was paired before in the image.  So group g's pair comes from the
// id of g's first feature k0 in the image: (the last feature with that id, g), and the pairs are in the order of k0.
// One block per image, features k = 16 * thread + i (blocked): a radix sort of (group << 13 | k) puts each group's features in
// feature order, a max-scan of the segment heads finds every feature's k0, and the features with k0's id raise its last index.
constexpr int kAssignThreads = 512, kAssignItems = 16, kAssignBits = 13;
static_assert(kAssignThreads * kAssignItems == OPB_SFM_ASSIGN_MAX_CAP && (1 << kAssignBits) == OPB_SFM_ASSIGN_MAX_CAP, "assign tile");
using AssignSort = cub::BlockRadixSort<uint64_t, kAssignThreads, kAssignItems>;
using AssignScan = cub::BlockScan<int, kAssignThreads>;
struct AssignSmem {
  union {
    typename AssignSort::TempStorage sort;
    uint64_t keys[OPB_SFM_ASSIGN_MAX_CAP];      // the sorted keys
  } a;
  typename AssignScan::TempStorage scan;
  int32_t rank[OPB_SFM_ASSIGN_MAX_CAP];         // feature k: its id's index among the kept ids, -1 without a kept id
  int32_t group[OPB_SFM_ASSIGN_MAX_CAP];        // at a group's first feature k0: the group
  int32_t last[OPB_SFM_ASSIGN_MAX_CAP];         // at k0: the last feature with k0's id; -1 elsewhere
};
constexpr uint64_t kNoKey = ~0ull;

__global__ void __launch_bounds__(kAssignThreads) assign_pairs_kernel(const int64_t* __restrict__ point3d_ids,
                                                                      const int32_t* __restrict__ counts, int cap,
                                                                      const int64_t* __restrict__ kept_ids,
                                                                      const int32_t* __restrict__ kept_group, int M, int end_bit,
                                                                      int64_t* __restrict__ packed, int64_t* __restrict__ num_matches) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  AssignSmem& sm = *reinterpret_cast<AssignSmem*>(smem_raw);
  const int f = blockIdx.x, n = min(counts[f], cap);
  uint64_t key[kAssignItems];
  for (int i = 0; i < kAssignItems; ++i) {
    const int k = threadIdx.x * kAssignItems + i;
    int32_t rank = -1;
    key[i] = kNoKey;
    if (k < n) {
      const int64_t id = point3d_ids[(size_t)f * cap + k];
      int lo = 0, hi = M;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (kept_ids[mid] < id) lo = mid + 1;
        else hi = mid;
      }
      if (id != -1 && lo < M && kept_ids[lo] == id) {
        rank = lo;
        key[i] = (uint64_t)kept_group[lo] << kAssignBits | (uint64_t)k;
      }
    }
    sm.rank[k] = rank;
    sm.last[k] = -1;
  }
  __syncthreads();
  AssignSort(sm.a.sort).Sort(key, 0, end_bit);
  __syncthreads();
  for (int i = 0; i < kAssignItems; ++i) sm.a.keys[threadIdx.x * kAssignItems + i] = key[i];
  __syncthreads();
  int head[kAssignItems];
  for (int i = 0; i < kAssignItems; ++i) {
    const int p = threadIdx.x * kAssignItems + i;
    head[i] = key[i] != kNoKey && (p == 0 || sm.a.keys[p - 1] >> kAssignBits != key[i] >> kAssignBits) ? p : -1;
  }
  AssignScan(sm.scan).InclusiveScan(head, head, cub::Max());
  for (int i = 0; i < kAssignItems; ++i) {
    if (key[i] == kNoKey) continue;
    const int p = threadIdx.x * kAssignItems + i;
    const int k = (int)(key[i] & (OPB_SFM_ASSIGN_MAX_CAP - 1)), k0 = (int)(sm.a.keys[head[i]] & (OPB_SFM_ASSIGN_MAX_CAP - 1));
    if (p == head[i]) sm.group[k0] = (int32_t)(key[i] >> kAssignBits);
    if (sm.rank[k] == sm.rank[k0]) atomicMax(&sm.last[k0], k);
  }
  __syncthreads();
  int slot[kAssignItems], total;
  for (int i = 0; i < kAssignItems; ++i) slot[i] = sm.last[threadIdx.x * kAssignItems + i] >= 0;
  AssignScan(sm.scan).ExclusiveSum(slot, slot, total);
  for (int i = 0; i < kAssignItems; ++i) {
    const int k = threadIdx.x * kAssignItems + i;
    if (sm.last[k] >= 0) packed[(size_t)f * cap + slot[i]] = (int64_t)sm.last[k] << 32 | sm.group[k];
  }
  if (threadIdx.x == 0) num_matches[f] = total;
}

// offsets[0 .. F] of the images' pairs (one thread: F is the number of images)
__global__ void assign_offsets_kernel(const int64_t* __restrict__ num_matches, int F, int64_t* __restrict__ offsets) {
  int64_t s = 0;
  for (int f = 0; f < F; ++f) {
    offsets[f] = s;
    s += num_matches[f];
  }
  offsets[F] = s;
}

// Image f's pairs from its padded row to columns offsets[f] .. of pairs [2, pair_stride]: the feature, then the group.
__global__ void assign_compact_kernel(const int64_t* __restrict__ packed, const int64_t* __restrict__ num_matches,
                                      const int64_t* __restrict__ offsets, int cap, int64_t pair_stride, int64_t* __restrict__ pairs) {
  const int f = blockIdx.x;
  const int64_t o = offsets[f];
  for (int i = threadIdx.x; i < num_matches[f]; i += blockDim.x) {
    const int64_t v = packed[(size_t)f * cap + i];
    pairs[o + i] = v >> 32;
    pairs[pair_stride + o + i] = v & 0xffffffff;
  }
}

// Workspace of opb_sfm_filter_points: the sorted lengths, then CUB's temporary storage.
int filter_temp_bytes(int P, size_t* bytes) {
  *bytes = 0;
  return cub::DeviceRadixSort::SortKeys(nullptr, *bytes, (const int64_t*)nullptr, (int64_t*)nullptr, P) == cudaSuccess ? 0 : -1;
}

// Workspace of opb_sfm_gather_observations: keys, values and their sorted copies [F * cap] int32 each, the per-slot counts
// [kept_cap] int32, then CUB's temporary storage.
int gather_temp_bytes(int64_t items, size_t* bytes) {
  *bytes = 0;
  return cub::DeviceRadixSort::SortPairs(nullptr, *bytes, (const int32_t*)nullptr, (int32_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr,
                                         (int)items) == cudaSuccess ? 0 : -1;
}

}  // namespace
}  // namespace opb

extern "C" int opb_sfm_filter_workspace_bytes(int32_t P, int64_t* bytes) {
  REQUIRE(__func__, bytes && P > 0);
  size_t tmp;
  if (opb::filter_temp_bytes(P, &tmp)) return opb::fail(opb::no_handle_error, OPB_E_CUDA, "%s: CUB size query failed", __func__);
  *bytes = (int64_t)(opb::align256((size_t)P * 8) + tmp);
  return OPB_OK;
}

extern "C" int opb_sfm_filter_points(const int64_t* ids, const double* xyz, const int64_t* track_len, int32_t P, int32_t max_num_kp3d,
                                     const double* corners, void* workspace, int64_t workspace_bytes, int64_t* kept_ids, float* kept_xyz,
                                     int64_t* track_length, int64_t* n_kept, void* stream) {
  REQUIRE(__func__, ids && xyz && track_len && corners && workspace && kept_ids && kept_xyz && track_length && n_kept);
  REQUIRE(__func__, P > 0 && max_num_kp3d >= 0);
  REQUIRE(__func__, ((uintptr_t)workspace & 255) == 0);
  size_t tmp;
  if (opb::filter_temp_bytes(P, &tmp)) return opb::fail(opb::no_handle_error, OPB_E_CUDA, "%s: CUB size query failed", __func__);
  const size_t sorted_bytes = opb::align256((size_t)P * 8);
  REQUIRE(__func__, workspace_bytes >= (int64_t)(sorted_bytes + tmp));
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* sorted = (int64_t*)workspace;
  const cudaError_t e = cub::DeviceRadixSort::SortKeys((char*)workspace + sorted_bytes, tmp, track_len, sorted, P, 0, 64, st);
  if (e != cudaSuccess) return opb::fail(opb::no_handle_error, OPB_E_CUDA, "%s: radix sort failed: %s", __func__, cudaGetErrorString(e));
  const int k0 = max(P - 1 - max_num_kp3d, 0);
  LAUNCH_NH(__func__, opb::filter_kernel, 1, opb::kFilterThreads, 0, st, xyz, track_len, ids, P, (const int64_t*)sorted, k0, corners, kept_ids,
            kept_xyz, track_length, n_kept);
  return OPB_OK;
}

extern "C" int opb_sfm_merge_workspace_bytes(int32_t cap, int64_t* bytes) {
  REQUIRE(__func__, bytes && cap > 0);
  *bytes = (int64_t)(2 * opb::align256((size_t)cap * 4));
  return OPB_OK;
}

extern "C" int opb_sfm_merge_points(const float* xyz, const int64_t* ids, const int64_t* n, int32_t cap, double dist_threshold, void* workspace,
                                    int64_t workspace_bytes, double* merged_xyz, int32_t* group_offsets, int64_t* member_ids, int32_t* member_index,
                                    int32_t* slot_of, int64_t* n_groups, int64_t* n_members, void* stream) {
  REQUIRE(__func__, xyz && ids && n && workspace && merged_xyz && group_offsets && member_ids && member_index && slot_of && n_groups &&
                        n_members);
  REQUIRE(__func__, cap > 0 && dist_threshold > 0.0);
  REQUIRE(__func__, ((uintptr_t)workspace & 255) == 0);
  const size_t part = opb::align256((size_t)cap * 4);
  REQUIRE(__func__, workspace_bytes >= (int64_t)(2 * part));
  int32_t* count = (int32_t*)workspace;
  int32_t* recorded = (int32_t*)((char*)workspace + part);
  cudaStream_t st = (cudaStream_t)stream;
  LAUNCH_NH(__func__, opb::neighbour_count_kernel, (unsigned)((cap + opb::kWarpsPerBlock - 1) / opb::kWarpsPerBlock), 32 * opb::kWarpsPerBlock, 0,
            st, xyz, n, cap, dist_threshold, count);
  LAUNCH_NH(__func__, opb::merge_greedy_kernel, 1, 32, 0, st, xyz, ids, n, cap, dist_threshold, (const int32_t*)count, recorded, merged_xyz,
            group_offsets, member_index, member_ids, slot_of, n_groups, n_members);
  return OPB_OK;
}

extern "C" int opb_sfm_gather_workspace_bytes(int32_t F, int32_t cap, int32_t kept_cap, int64_t* bytes) {
  REQUIRE(__func__, bytes && F > 0 && cap > 0 && kept_cap > 0 && (int64_t)F * cap <= (int64_t)INT32_MAX);
  const int64_t items = (int64_t)F * cap;
  size_t tmp;
  if (opb::gather_temp_bytes(items, &tmp)) return opb::fail(opb::no_handle_error, OPB_E_CUDA, "%s: CUB size query failed", __func__);
  *bytes = (int64_t)(4 * opb::align256((size_t)items * 4) + opb::align256((size_t)kept_cap * 4) + tmp);
  return OPB_OK;
}

extern "C" int opb_sfm_gather_observations(const int64_t* point3d_ids, const int32_t* counts, int32_t F, int32_t cap, const int64_t* kept_ids,
                                           const int64_t* n_kept, int32_t kept_cap, const int32_t* slot_of, const int32_t* group_offsets,
                                           const int64_t* n_groups, void* workspace, int64_t workspace_bytes, int32_t* order, int64_t* idxs,
                                           int64_t* total, int64_t* missing, void* stream) {
  REQUIRE(__func__, point3d_ids && counts && kept_ids && n_kept && slot_of && group_offsets && n_groups && workspace && order && idxs && total &&
                        missing);
  REQUIRE(__func__, F > 0 && cap > 0 && kept_cap > 0 && (int64_t)F * cap <= (int64_t)INT32_MAX);
  REQUIRE(__func__, ((uintptr_t)workspace & 255) == 0);
  const int64_t items = (int64_t)F * cap;
  size_t tmp;
  if (opb::gather_temp_bytes(items, &tmp)) return opb::fail(opb::no_handle_error, OPB_E_CUDA, "%s: CUB size query failed", __func__);
  const size_t part = opb::align256((size_t)items * 4);
  REQUIRE(__func__, workspace_bytes >= (int64_t)(4 * part + opb::align256((size_t)kept_cap * 4) + tmp));
  char* w = (char*)workspace;
  int32_t* keys = (int32_t*)w;
  int32_t* vals = (int32_t*)(w + part);
  int32_t* keys_sorted = (int32_t*)(w + 2 * part);
  int32_t* vals_sorted = (int32_t*)(w + 3 * part);
  int32_t* slot_count = (int32_t*)(w + 4 * part);
  void* cub_tmp = w + 4 * part + opb::align256((size_t)kept_cap * 4);
  cudaStream_t st = (cudaStream_t)stream;
  CK(opb::no_handle_error, cudaMemsetAsync(slot_count, 0, (size_t)kept_cap * 4, st));
  CK(opb::no_handle_error, cudaMemsetAsync(total, 0, 8, st));
  CK(opb::no_handle_error, cudaMemsetAsync(missing, 0x7f, 8, st));   // above every slot: no member without an observation
  LAUNCH_NH(__func__, opb::observation_keys_kernel, (unsigned)((items + 255) / 256), 256, 0, st, point3d_ids, counts, F, cap, kept_ids, n_kept,
            kept_cap, slot_of, keys, vals, slot_count);
  // a stable sort on the slot: within a slot the features stay in (image, feature) order; kNoSlot sorts last
  const cudaError_t e = cub::DeviceRadixSort::SortPairs(cub_tmp, tmp, keys, keys_sorted, vals, vals_sorted, (int)items, 0, 31, st);
  if (e != cudaSuccess) return opb::fail(opb::no_handle_error, OPB_E_CUDA, "%s: radix sort failed: %s", __func__, cudaGetErrorString(e));
  CK(opb::no_handle_error, cudaMemcpyAsync(order, vals_sorted, (size_t)items * 4, cudaMemcpyDeviceToDevice, st));
  LAUNCH_NH(__func__, opb::group_counts_kernel, (unsigned)((kept_cap + 255) / 256), 256, 0, st, group_offsets, n_groups, kept_cap,
            (const int32_t*)slot_count, idxs, (unsigned long long*)total, missing);
  return OPB_OK;
}

extern "C" int opb_sfm_gather_features(const int32_t* order, int64_t total, int32_t F, int32_t cap, int32_t D, const float* scores,
                                       const float* descriptors, double* out_descriptors, double* out_scores, void* stream) {
  REQUIRE(__func__, total >= 0 && F > 0 && cap > 0 && D > 0 && total <= (int64_t)F * cap && total <= (int64_t)INT32_MAX);
  REQUIRE(__func__, total == 0 || (order && scores && descriptors && out_descriptors && out_scores));
  if (total > 0)
    LAUNCH_NH(__func__, opb::gather_features_kernel, (unsigned)total, 128, 0, (cudaStream_t)stream, order, total, cap, D, scores, descriptors,
              out_descriptors, out_scores);
  return OPB_OK;
}

extern "C" int opb_sfm_assign_workspace_bytes(int32_t F, int32_t cap, int64_t* bytes) {
  REQUIRE(__func__, bytes && F > 0 && cap > 0 && cap <= OPB_SFM_ASSIGN_MAX_CAP && (int64_t)F * cap <= (int64_t)INT32_MAX);
  *bytes = (int64_t)opb::align256((size_t)F * cap * 8);
  return OPB_OK;
}

extern "C" int opb_sfm_assign_pairs(const int64_t* point3d_ids, const int32_t* counts, int32_t F, int32_t cap, const int64_t* kept_ids,
                                    const int32_t* kept_group, int32_t M, void* workspace, int64_t workspace_bytes, int64_t* pairs,
                                    int64_t* offsets, int64_t* num_matches, void* stream) {
  REQUIRE(__func__, point3d_ids && counts && kept_ids && kept_group && workspace && pairs && offsets && num_matches);
  REQUIRE(__func__, F > 0 && cap > 0 && cap <= OPB_SFM_ASSIGN_MAX_CAP && M > 0 && (int64_t)F * cap <= (int64_t)INT32_MAX);
  REQUIRE(__func__, ((uintptr_t)workspace & 255) == 0);
  REQUIRE(__func__, workspace_bytes >= (int64_t)opb::align256((size_t)F * cap * 8));
  int group_bits = 0;                   // groups are below M: below the all-ones key of a feature without a kept id
  while (group_bits < 31 && (1ll << group_bits) <= (int64_t)M) ++group_bits;
  const size_t smem = sizeof(opb::AssignSmem);
  CK(opb::no_handle_error, cudaFuncSetAttribute(opb::assign_pairs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* packed = (int64_t*)workspace;
  LAUNCH_NH(__func__, opb::assign_pairs_kernel, (unsigned)F, opb::kAssignThreads, smem, st, point3d_ids, counts, (int)cap, kept_ids, kept_group,
            (int)M, opb::kAssignBits + group_bits, packed, num_matches);
  LAUNCH_NH(__func__, opb::assign_offsets_kernel, 1, 1, 0, st, (const int64_t*)num_matches, (int)F, offsets);
  LAUNCH_NH(__func__, opb::assign_compact_kernel, (unsigned)F, 256, 0, st, (const int64_t*)packed, (const int64_t*)num_matches,
            (const int64_t*)offsets, (int)cap, (int64_t)F * cap, pairs);
  return OPB_OK;
}
