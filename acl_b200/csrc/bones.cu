// acl_b200/csrc/bones.cu -- the bone query (aclb200_decompress_bones): chosen bones of each pose, in local or object space, decoding and
// walking only the ancestor chains of the requested bones.
//
// A request names a list of up to 32 bones. Its row j is byte for byte row list[j] of what aclb200_decompress_tracks (no parents) or
// aclb200_decompress_tracks_object_space (parents) computes for the request: the decode is the plain kernel's decode restricted to some
// bones (decode_bone_row: the plain kernel's decoders, SINGLE = false), and the walk is object_space.cuh's walk restricted to an
// ancestor-closed set of bones (pose_rows_to_object_space<CLOSURE = true>), whose rows never read a bone outside the set.
//
// Work decomposition, thread block = `requests_per_block` whole requests (BoneQuery::requests_per_block):
//   bone_query_block (bone_closure.cuh, shared with the pose features) with BoneRowsStage:
//   phase 1  one thread per request: the seek (seek_transform) and the request's list index, into shared memory.
//   phases 2 to 4  each request's ancestor closure is marked, listed, decoded (decode_bone_row) and, with parents, walked to object space.
//   phase 5  the listed rows leave shared memory as coalesced 16 byte (QVV48) or 8 byte (QVV40) stores.
#include "bone_closure.cuh"

#include <type_traits>

namespace aclb200
{
	using namespace dev;

	namespace
	{
		constexpr uint32_t k_bones_target_requests = 8;				// one request per warp of the walk
		constexpr uint32_t k_bones_block_budget = 48u * 1024u;		// up to 4 blocks of 8 C2 requests per SM

		// phase 1 and phase 5 of the bone query's block (bone_closure.cuh)
		template<bool DB>
		struct BoneRowsStage
		{
			// ---- phase 1: the seek (seek_transform) and the request's list index; a list index >= num_lists writes nothing ----
			template<class RS>
			__device__ __forceinline__ void seek(const DecodeParams& p, const BoneQuery& q, uint32_t first_request, RS* s_req, uint32_t* s_words) const
			{
				RS rs;
				seek_transform<DB>(p, first_request + threadIdx.x, rs);
				const uint32_t list = q.request_lists != nullptr ? __ldg(q.request_lists + first_request + threadIdx.x) : 0u;
				if (list >= q.num_lists)
					rs.num_tracks = 0;
				s_req[threadIdx.x] = rs;
				s_words[threadIdx.x * 4] = rs.num_tracks != 0 ? list : k_no_list;
			}

			template<class RS>
			__device__ __forceinline__ void before_closures(const DecodeParams&, const RS*, const uint32_t*, uint32_t, uint32_t) const {}

			// ---- phase 5: row j of request r is row list[j] of its pose rows; 16 byte chunks (QVV48) or 8 byte chunks (QVV40) ----
			template<class RS>
			__device__ __forceinline__ void finish(const DecodeParams& p, const BoneQuery& q, const RS* s_req, const uint32_t* s_words,
				const uint8_t* s_pose, uint32_t first_request, uint32_t num_requests) const
			{
				__syncthreads();
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
		};

		template<int NORM, bool PER_TRACK, bool DB>
		__global__ void __launch_bounds__(k_threads_per_block)
		transform_decompress_bones_kernel(const DecodeParams p, const BoneQuery q)
		{
			bone_query_block<NORM, PER_TRACK, DB>(p, q, BoneRowsStage<DB>{});
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
	bool plan_bones_launch(const DecodeParams& params, BoneQuery& query, bool database, int max_dynamic_smem, uint32_t extra_request_bytes)
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
			const uint64_t bytes = query.smem_pose_offset + uint64_t(requests) * (uint64_t(query.smem_pose_bytes) + extra_request_bytes);
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
