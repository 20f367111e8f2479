// acl_b200/csrc/bones.cu -- the bone query (aclb200_decompress_bones): chosen bones of each pose, in local or object space, decoding and
// walking only the ancestor chains of the requested bones.
//
// A request names a list of up to 32 bones. Its row j is byte for byte row list[j] of what aclb200_decompress_tracks (no parents) or
// aclb200_decompress_tracks_object_space (parents) computes for the request: the decode is the plain kernel's decode restricted to some
// bones (decode_bone_row: the plain kernel's decoders, SINGLE = false), and the walk is object_space.cuh's walk restricted to an
// ancestor-closed set of bones (pose_rows_to_object_space<CLOSURE = true>), whose rows never read a bone outside the set.
//
// Work decomposition, thread block = `requests_per_block` whole requests (BoneQuery::requests_per_block):
//   phase 1  one thread per request: the seek (seek_transform) and the request's list index, into shared memory.
//   phase 2  one warp per request, one lane per list entry: the lane walks its bone's parents and ORs them into the request's closure
//            bitmask (max_tracks bits). It stops at a root, at a parent that does not precede its child, or at a bone another lane has
//            already marked (that lane walks on from there). Without parents the closure is the listed bones. The warp then compacts the
//            closure into the block's (request, bone) work list.
//   phase 3  one thread per (request, closure bone): decode_bone_row, the constant, default and animated sub-tracks of the bone with key
//            frames read from global memory (a query touches a few sub-tracks of each key frame), into the bone's row of the request's
//            pose rows.
//   phase 4  with parents: one warp per request walks the closure bones (wavefronts of 32 bones, chunks without a closure bone skipped).
//   phase 5  the listed rows leave shared memory as coalesced 16 byte (QVV48) or 8 byte (QVV40) stores.
#include "device_common.cuh"
#include "object_space.cuh"

#include <type_traits>

namespace aclb200
{
	using namespace dev;

	namespace
	{
		constexpr uint32_t k_bones_target_requests = 8;				// one request per warp of the walk
		constexpr uint32_t k_bones_block_budget = 48u * 1024u;		// up to 4 blocks of 8 C2 requests per SM
		constexpr uint32_t k_item_bone_bits = 26;					// a work item: bone | local request << 26 (64 requests, 2^26 bones)
		static_assert(k_max_tracks <= (1u << k_item_bone_bits) && k_max_requests_per_block <= 64, "a work item holds a bone and a request");

		// per request words beside the request states: [0] the list index (k_no_list: the request writes nothing), [1] the first work item
		// of the request, [2] its closure size
		constexpr uint32_t k_no_list = 0xFFFFFFFFu;

		template<int NORM, bool PER_TRACK, bool DB>
		__global__ void __launch_bounds__(k_threads_per_block)
		transform_decompress_bones_kernel(const DecodeParams p, const BoneQuery q)
		{
			using RS = typename std::conditional<DB, ReqStateDB, ReqState>::type;
			// dynamic shared memory: RS[requests_per_block] | request words u32[requests_per_block][4] | closure bitmasks
			// u32[requests_per_block][mask_words] | work items u32[requests_per_block * max_tracks] | pose rows
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
			{
				RS rs;
				seek_transform<DB>(p, first_request + threadIdx.x, rs);
				const uint32_t list = q.request_lists != nullptr ? __ldg(q.request_lists + first_request + threadIdx.x) : 0u;
				if (list >= q.num_lists)
					rs.num_tracks = 0;
				s_req[threadIdx.x] = rs;
				s_words[threadIdx.x * 4] = rs.num_tracks != 0 ? list : k_no_list;
			}
			for (uint32_t word = threadIdx.x; word < num_requests * q.mask_words; word += k_threads_per_block)
				s_mask[word] = 0;
			__syncthreads();

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

			// ---- phase 5: row j of request r is row list[j] of its pose rows; 16 byte chunks (QVV48) or 8 byte chunks (QVV40) ----
			__syncthreads();
			{
				const bool qvv40 = p.layout == ACLB200_LAYOUT_QVV40;
				const uint32_t chunk_bytes = qvv40 ? 8u : 16u;
				const uint32_t chunks_per_row = p.bone_stride / chunk_bytes;
				const uint32_t chunks_per_request = q.bones_per_list * chunks_per_row;
				const uint32_t num_chunks = num_requests * chunks_per_request;
				for (uint32_t slot = threadIdx.x; slot < num_chunks; slot += k_threads_per_block)
				{
					const uint32_t local_request = slot / chunks_per_request;
					const uint32_t in_request = slot - local_request * chunks_per_request;
					const uint32_t entry = in_request / chunks_per_row;
					const uint32_t chunk = in_request - entry * chunks_per_row;
					const uint32_t list = s_words[local_request * 4];
					if (list == k_no_list)
						continue;
					const uint32_t bone = __ldg(q.bone_lists + size_t(list) * q.bones_per_list + entry);
					if (bone >= s_req[local_request].num_tracks)
						continue;		// ACLB200_NO_BONE, or a bone the clip does not have: the row is left as it is
					const uint8_t* src = s_pose + size_t(local_request) * q.smem_pose_bytes + size_t(bone) * p.bone_stride + chunk * chunk_bytes;
					uint8_t* dst = p.out + uint64_t(first_request + local_request) * p.pose_stride + entry * p.bone_stride + chunk * chunk_bytes;
					if (qvv40)
						*reinterpret_cast<uint2*>(dst) = *reinterpret_cast<const uint2*>(src);
					else
						*reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
				}
			}
		}

		using BonesKernel = void (*)(DecodeParams, BoneQuery);

		BonesKernel bones_kernel(uint32_t normalization, bool per_track, bool database)
		{
			return with_constant<3>(normalization, [&](auto NORM) { return with_bool(per_track, [&](auto PER_TRACK) {
				return with_bool(database, [&](auto DB) -> BonesKernel { return transform_decompress_bones_kernel<NORM, PER_TRACK, DB>; }); }); });
		}
	}

	cudaError_t configure_bones_kernels(int max_dynamic_smem)
	{
		cudaError_t error = cudaSuccess;
		for (uint32_t choice = 0; choice < 12 && error == cudaSuccess; ++choice)
			error = cudaFuncSetAttribute(bones_kernel(choice / 4, (choice & 1) != 0, (choice & 2) != 0), cudaFuncAttributeMaxDynamicSharedMemorySize,
				max_dynamic_smem);
		return error;
	}

	// Up to 8 requests per block within 48 KB, at least one within the whole budget: max_tracks pose rows per request, as the object space
	// decode plans them, plus the closure bitmask, the request's share of the work list and its state
	bool plan_bones_launch(const DecodeParams& params, BoneQuery& query, bool database, int max_dynamic_smem)
	{
		const uint32_t max_tracks = params.max_tracks == 0 ? 1 : params.max_tracks;
		const uint32_t state_bytes = database ? uint32_t(sizeof(ReqStateDB)) : uint32_t(sizeof(ReqState));
		query.mask_words = (max_tracks + 31) / 32;
		query.smem_pose_bytes = (max_tracks * params.bone_stride + 15) & ~15u;
		const auto lay_out = [&](uint32_t requests)
		{
			query.requests_per_block = requests;
			query.smem_words_offset = requests * state_bytes;
			query.smem_mask_offset = (query.smem_words_offset + requests * 16 + 15) & ~15u;
			query.smem_items_offset = query.smem_mask_offset + requests * query.mask_words * 4;
			query.smem_pose_offset = (query.smem_items_offset + requests * max_tracks * 4 + 15) & ~15u;
			const uint64_t bytes = query.smem_pose_offset + uint64_t(requests) * query.smem_pose_bytes;
			query.smem_bytes = uint32_t(bytes < 0xFFFFFFFFu ? bytes : 0xFFFFFFFFu);
			return bytes;
		};
		uint32_t requests_per_block = k_bones_target_requests;
		while (requests_per_block > 1 && lay_out(requests_per_block) > k_bones_block_budget)
			--requests_per_block;
		return lay_out(requests_per_block) <= uint64_t(max_dynamic_smem > 0 ? max_dynamic_smem : 0);
	}

	cudaError_t launch_decompress_bones(const DecodeParams& params, const BoneQuery& query, bool database, cudaStream_t stream)
	{
		const uint32_t blocks = (params.num_requests + query.requests_per_block - 1) / query.requests_per_block;
		bones_kernel(params.normalization, params.per_track_rounding != 0, database)<<<blocks, k_threads_per_block, query.smem_bytes, stream>>>(params, query);
		return cudaGetLastError();
	}
}
