// acl_b200/csrc/bone_closure.cuh -- one block of the bone query (bones.cu) and of the pose features (features.cu): the bone query's plan,
// which decodes and walks the ancestor closure of each request's bone list, with the steps that differ between the two supplied by a
// `Stage` (the bone query's BoneRowsStage in bones.cu, the pose features' FeatureStage in features.cu).
//
// Work decomposition, thread block = `requests_per_block` whole requests (BoneQuery::requests_per_block):
//   phase 1  one thread per request (request first_request + threadIdx.x): Stage::seek puts its seek state in s_req[threadIdx.x] and its
//            list index in word 0 of its request words (k_no_list, and num_tracks 0 in its state, when it writes nothing); the closure
//            bitmasks are cleared.
//   Stage::before_closures (after a block barrier)
//   phase 2  one warp per request, one lane per list entry: the lane walks its bone's parents and ORs them into the request's closure
//            bitmask (max_tracks bits). It stops at a root, at a parent that does not precede its child, or at a bone another lane has
//            already marked (that lane walks on from there). Without parents the closure is the listed bones. The warp then compacts the
//            closure into the block's (request, bone) work list.
//   phase 3  one thread per (request, closure bone): decode_bone_row, the constant, default and animated sub-tracks of the bone with key
//            frames read from global memory (a query touches a few sub-tracks of each key frame), into the bone's row of the request's
//            pose rows.
//   phase 4  with parents: one warp per request walks the closure bones (wavefronts of 32 bones, chunks without a closure bone skipped).
//   Stage::finish (no barrier before it): the rows leave.
// The block is one function that the kernels inline whole, and Stage::seek does all of phase 1 for its thread: a function for phases 2
// to 4 alone, or a seek hook that returned the list index to the block, changed the bone query's SASS (register allocation and
// scheduling); this form compiles to the SASS of the bone query's former single kernel body.
#pragma once

#include "device_common.cuh"
#include "object_space.cuh"

#include <type_traits>

namespace aclb200
{
	namespace dev
	{
		constexpr uint32_t k_item_bone_bits = 26;					// a work item: bone | local request << 26 (64 requests, 2^26 bones)
		static_assert(k_max_tracks <= (1u << k_item_bone_bits) && k_max_requests_per_block <= 64, "a work item holds a bone and a request");

		// per request words beside the request states: [0] the list index (k_no_list: the request writes nothing), [1] the first work item
		// of the request, [2] its closure size
		constexpr uint32_t k_no_list = 0xFFFFFFFFu;

		// The shared memory of a block: RS[requests_per_block] | request words u32[requests_per_block][4] | closure bitmasks
		// u32[requests_per_block][mask_words] | work items u32[requests_per_block * max_tracks] | pose rows (| the stage's own bytes per
		// request, plan_bones_launch's extra_request_bytes)
		template<int NORM, bool PER_TRACK, bool DB, class Stage>
		__device__ __forceinline__ void bone_query_block(const DecodeParams& p, const BoneQuery& q, const Stage& stage)
		{
			using RS = typename std::conditional<DB, ReqStateDB, ReqState>::type;
			extern __shared__ __align__(16) uint8_t s_dynamic[];
			RS* s_req = reinterpret_cast<RS*>(s_dynamic);
			uint32_t* s_words = reinterpret_cast<uint32_t*>(s_dynamic + q.smem_words_offset);
			uint32_t* s_mask = reinterpret_cast<uint32_t*>(s_dynamic + q.smem_mask_offset);
			uint32_t* s_items = reinterpret_cast<uint32_t*>(s_dynamic + q.smem_items_offset);
			uint8_t* s_pose = s_dynamic + q.smem_pose_offset;

			const uint32_t first_request = blockIdx.x * q.requests_per_block;
			const uint32_t num_requests = min(q.requests_per_block, p.num_requests - first_request);
			const uint32_t lane = threadIdx.x & 31u;
			const uint32_t warp = threadIdx.x >> 5;

			// ---- phase 1: seek, list index; the closure bitmasks are cleared ----
			if (threadIdx.x < num_requests)
				stage.seek(p, q, first_request, s_req, s_words);
			for (uint32_t word = threadIdx.x; word < num_requests * q.mask_words; word += k_threads_per_block)
				s_mask[word] = 0;
			__syncthreads();
			stage.before_closures(p, s_req, s_words, first_request, num_requests);

			// ---- phase 2: one warp per request marks the ancestor closure of its listed bones, counts it ----
			for (uint32_t local_request = warp; local_request < num_requests; local_request += k_threads_per_block / 32)
			{
				const uint32_t list = s_words[local_request * 4];
				uint32_t* mask = s_mask + local_request * q.mask_words;
				uint32_t count = 0;
				if (list != k_no_list)
				{
					const uint32_t num_tracks = s_req[local_request].num_tracks;
					const uint32_t* parents = nullptr;
					if (q.parent_indices != nullptr)
						parents = q.parent_indices + (q.skeleton_offsets != nullptr ? __ldg(q.skeleton_offsets + s_req[local_request].clip) : 0u);
					uint32_t bone = lane < q.bones_per_list ? __ldg(q.bone_lists + size_t(list) * q.bones_per_list + lane) : obj::k_invalid_track;
					// a walk only ever moves to a parent strictly below its bone: it ends on any parent table
					while (bone < num_tracks)
					{
						const uint32_t bit = 1u << (bone & 31u);
						if ((atomicOr(mask + (bone >> 5), bit) & bit) != 0 || parents == nullptr)
							break;
						const uint32_t parent = __ldg(parents + bone);
						bone = parent < bone ? parent : obj::k_invalid_track;
					}
					__syncwarp();
					for (uint32_t word = lane; word < q.mask_words; word += 32)
						count += __popc(mask[word]);
					count = __reduce_add_sync(0xFFFFFFFFu, count);
				}
				if (lane == 0)
					s_words[local_request * 4 + 2] = count;
			}
			__syncthreads();

			// ---- the work list: request r's closure bones at items [first of r, first of r + count of r), in bone order ----
			for (uint32_t local_request = warp; local_request < num_requests; local_request += k_threads_per_block / 32)
			{
				uint32_t first = 0;
				for (uint32_t r = lane; r < local_request; r += 32)
					first += s_words[r * 4 + 2];
				first = __reduce_add_sync(0xFFFFFFFFu, first);
				if (lane == 0)
					s_words[local_request * 4 + 1] = first;
				if (s_words[local_request * 4 + 2] == 0)
					continue;
				const uint32_t* mask = s_mask + local_request * q.mask_words;
				for (uint32_t word_index = 0; word_index < q.mask_words; ++word_index)
				{
					const uint32_t word = mask[word_index];
					if (((word >> lane) & 1u) != 0)
						s_items[first + __popc(word & ((1u << lane) - 1u))] = (word_index * 32 + lane) | (local_request << k_item_bone_bits);
					first += __popc(word);
				}
			}
			__syncthreads();

			// ---- phase 3: one thread per (request, closure bone) decodes the bone's three sub-tracks into its row ----
			{
				const uint32_t last = num_requests - 1;
				const uint32_t num_items = s_words[last * 4 + 1] + s_words[last * 4 + 2];
				for (uint32_t item = threadIdx.x; item < num_items; item += k_threads_per_block)
				{
					const uint32_t packed = s_items[item];
					const uint32_t local_request = packed >> k_item_bone_bits;
					const uint32_t bone = packed & ((1u << k_item_bone_bits) - 1u);
					decode_bone_row<NORM, PER_TRACK>(p, s_req[local_request], bone,
						s_pose + size_t(local_request) * q.smem_pose_bytes + size_t(bone) * p.bone_stride);
				}
			}

			// ---- phase 4: one warp per request takes its closure rows to object space ----
			if (q.parent_indices != nullptr)
			{
				__syncthreads();
				uint32_t flags = 0;
				for (uint32_t local_request = warp; local_request < num_requests; local_request += k_threads_per_block / 32)
				{
					if (s_words[local_request * 4 + 2] == 0)
						continue;
					const RS& rs = s_req[local_request];
					const uint32_t skeleton = q.skeleton_offsets != nullptr ? __ldg(q.skeleton_offsets + rs.clip) : 0u;
					flags |= obj::pose_rows_to_object_space<true>(s_pose + size_t(local_request) * q.smem_pose_bytes, rs.num_tracks,
						q.parent_indices + skeleton, q.object_kind != ACLB200_OBJECT_QVVF, s_mask + local_request * q.mask_words);
				}
				flags = __reduce_or_sync(0xFFFFFFFFu, flags);
				if (lane == 0 && flags != 0 && q.out_flags != nullptr)
					atomicOr(q.out_flags, flags);
			}

			stage.finish(p, q, s_req, s_words, s_pose, first_request, num_requests);
		}
	}
}
