// acl_b200/csrc/features.cu -- the pose features (aclb200_extract_pose_features): chosen bones of each request at up to eight time offsets,
// each in the root's frame at the request's time, across loop boundaries.
//
// Each (request r, offset s) pair is a virtual request r * S + s with its own time u'. Virtual requests are independent (each decodes
// its own root samples), so the bone query's plan runs on them unchanged: up to 8 virtual requests per block, no block has to hold every
// offset of a request. Row (s, k) is F = qvv_mul(qvv_mul(B, qvv_inverse(T(u'))), M), where B is the bone query's object row of entry k at
// u', T the root's local row and M root motion's row for {clip, t, u', c}.
//
// Work decomposition, thread block = `requests_per_block` whole virtual requests (BoneQuery::requests_per_block):
//   phase 1  one thread per virtual request: the request's fields, the offset time u' and loop count c, the seek at u' and the list index.
//   samples  one thread per (virtual request, sample slot), as root motion's lanes: slot 0 t, slot 1 u', slot 2 the clamp duration D,
//            slot 3 time 0 (slots 2 and 3 only when c != 0). The thread seeks its own time and decodes the root (decode_bone_row) into
//            the virtual request's sample rows.
//   phases 2 to 4  the bone query's (bone_query_block, bone_closure.cuh, with FeatureStage): the closure of the list is marked, decoded
//            and walked to object space.
//   compose  one thread per virtual request: M (obj::compose_root_motion, root motion's composition) and qvv_inverse(T(u')).
//   rows     one thread per listed row: F, stored as a 48 byte qvvf row.
#include "bone_closure.cuh"

#include <type_traits>

namespace aclb200
{
	using namespace dev;

	namespace
	{
		using obj::Qvv;

		// the virtual request's state beside its pose rows: the root samples T(t), T(u'), T(D), T(0), then M and qvv_inverse(T(u'))
		struct FeatureSlot
		{
			float time;					// t
			float offset_time;			// u'
			int32_t cycles;				// c
			uint32_t root;
			float4 rows[6][3];
		};
		static_assert(sizeof(FeatureSlot) % 16 == 0, "feature slots keep the rows after them 16 byte aligned");
		constexpr uint32_t k_samples = 4;
		constexpr uint32_t k_motion_row = 4;
		constexpr uint32_t k_inverse_row = 5;

		// phase 1, the root samples and the rows of the pose features' block (bone_closure.cuh)
		template<int NORM, bool PER_TRACK, bool DB>
		struct FeatureStage
		{
			const FeatureQuery& f;
			FeatureSlot* s_slot;			// [requests_per_block], after the pose rows

			// ---- phase 1: the request, its offset time, the seek at u' and the list index ----
			template<class RS>
			__device__ __forceinline__ void seek(const DecodeParams& p, const BoneQuery& q, uint32_t first_request, RS* s_req, uint32_t* s_words) const
			{
				const uint32_t virtual_request = first_request + threadIdx.x;
				const uint32_t request = virtual_request / f.num_offsets;
				const float offset = f.offsets[virtual_request - request * f.num_offsets];
				// three 4 byte loads: the ABI only promises the request array the 4 byte alignment of its fields
				const uint32_t* fields = reinterpret_cast<const uint32_t*>(f.requests + request);
				const uint32_t clip_index = __ldg(fields);
				const float time = __uint_as_float(__ldg(fields + 1));
				const uint32_t looping = __ldg(fields + 2);
				const uint32_t list = q.request_lists != nullptr ? __ldg(q.request_lists + request) : 0u;
				bool writes = false;
				uint32_t root = 0;
				int32_t cycles = 0;
				float offset_time = 0.0f;
				if (clip_index < p.num_clips && list < q.num_lists && looping <= ACLB200_FEATURE_LOOP)
				{
					const ClipDesc& clip = p.clips[clip_index];
					root = f.root_tracks != nullptr ? __ldg(f.root_tracks + clip_index) : 0u;
					offset_time = __fadd_rn(time, offset);
					writes = root < clip.num_tracks;
					if (looping == ACLB200_FEATURE_LOOP)
					{
						const float duration = clip.duration_clamp;
						if (!isfinite(offset_time))
							writes = false;
						else if (duration == 0.0f)
							offset_time = 0.0f;
						else
						{
							const float cycle = floorf(__fdiv_rn(offset_time, duration));
							if (!(fabsf(cycle) <= float(ACLB200_MAX_ROOT_MOTION_CYCLES)))
								writes = false;
							else
							{
								cycles = int32_t(cycle);
								offset_time = __fsub_rn(offset_time, __fmul_rn(cycle, duration));
							}
						}
					}
				}
				RS rs;
				seek_request<DB>(p, aclb200_request{ writes ? clip_index : 0xFFFFFFFFu, offset_time }, virtual_request, rs);
				s_req[threadIdx.x] = rs;
				s_words[threadIdx.x * 4] = rs.num_tracks != 0 ? list : k_no_list;
				FeatureSlot& slot = s_slot[threadIdx.x];
				slot.time = time;
				slot.offset_time = offset_time;
				slot.cycles = cycles;
				slot.root = root;
			}

			// ---- the root samples: one thread per (virtual request, sample slot) decodes the root into the slot's row ----
			template<class RS>
			__device__ __forceinline__ void before_closures(const DecodeParams& p, const RS* s_req, const uint32_t* s_words, uint32_t first_request,
				uint32_t num_requests) const
			{
				for (uint32_t item = threadIdx.x; item < num_requests * k_samples; item += k_threads_per_block)
				{
					const uint32_t local_request = item / k_samples;
					const uint32_t sample = item - local_request * k_samples;
					const FeatureSlot& slot = s_slot[local_request];
					if (s_words[local_request * 4] == k_no_list || (sample >= 2 && slot.cycles == 0))
						continue;
					// each sample seeks its own time, T(u') included: decoding it from phase 1's state in s_req instead took that state through a
					// generic pointer, grew the stack frame from 536 to 672-720 B and made the C2 database build 3 % slower (H100)
					const uint32_t clip_index = s_req[local_request].clip;
					const float time = sample == 0 ? slot.time : sample == 1 ? slot.offset_time : sample == 2 ? p.clips[clip_index].duration_clamp : 0.0f;
					RS rs;
					seek_request<DB>(p, aclb200_request{ clip_index, time }, first_request + local_request, rs);
					decode_bone_row<NORM, PER_TRACK>(p, rs, slot.root, reinterpret_cast<uint8_t*>(s_slot[local_request].rows[sample]));
				}
			}

			template<class RS>
			__device__ __forceinline__ void finish(const DecodeParams& p, const BoneQuery& q, const RS* s_req, const uint32_t* s_words,
				const uint8_t* s_pose, uint32_t first_request, uint32_t num_requests) const
			{
				__syncthreads();

				// ---- compose: M and the inverse of T(u') of each virtual request ----
				uint32_t flags = 0;
				if (threadIdx.x < num_requests && s_words[threadIdx.x * 4] != k_no_list)
				{
					FeatureSlot& slot = s_slot[threadIdx.x];
					const Qvv<float> to = obj::load_qvv_row(slot.rows[1]);
					const Qvv<float> motion = obj::compose_root_motion(obj::load_qvv_row(slot.rows[0]), to, obj::load_qvv_row(slot.rows[2]),
						obj::load_qvv_row(slot.rows[3]), slot.cycles, p.clips[s_req[threadIdx.x].clip].flags, flags);
					obj::store_qvv_row(slot.rows[k_motion_row], motion);
					obj::store_qvv_row(slot.rows[k_inverse_row], obj::qvv_inverse(to));
				}
				__syncthreads();

				// ---- rows: F = qvv_mul(qvv_mul(B, qvv_inverse(T(u'))), M) of each listed bone ----
				for (uint32_t row = threadIdx.x; row < num_requests * q.bones_per_list; row += k_threads_per_block)
				{
					const uint32_t local_request = row / q.bones_per_list;
					const uint32_t entry = row - local_request * q.bones_per_list;
					const uint32_t list = s_words[local_request * 4];
					if (list == k_no_list)
						continue;
					const uint32_t bone = __ldg(q.bone_lists + size_t(list) * q.bones_per_list + entry);
					if (bone >= s_req[local_request].num_tracks)
						continue;		// ACLB200_NO_BONE, or a bone the clip does not have: the row is left as it is
					const FeatureSlot& slot = s_slot[local_request];
					const Qvv<float> object = obj::load_qvv_row(reinterpret_cast<const float4*>(s_pose + size_t(local_request) * q.smem_pose_bytes
						+ size_t(bone) * p.bone_stride));
					const Qvv<float> relative = obj::flagged_qvv_mul(object, obj::load_qvv_row(slot.rows[k_inverse_row]), flags);
					const Qvv<float> feature = obj::flagged_qvv_mul(relative, obj::load_qvv_row(slot.rows[k_motion_row]), flags);
					const uint32_t virtual_request = first_request + local_request;
					const uint32_t request = virtual_request / f.num_offsets;
					const uint32_t offset = virtual_request - request * f.num_offsets;
					obj::store_qvv_row(reinterpret_cast<float4*>(p.out + uint64_t(request) * p.pose_stride
						+ (uint64_t(offset) * q.bones_per_list + entry) * 48), feature);
				}
				flags = __reduce_or_sync(0xFFFFFFFFu, flags);
				if ((threadIdx.x & 31u) == 0 && flags != 0 && q.out_flags != nullptr)
					atomicOr(q.out_flags, flags);
			}
		};

		// virtual request r * num_offsets + s is request r at offset s
		template<int NORM, bool PER_TRACK, bool DB>
		__global__ void __launch_bounds__(k_threads_per_block)
		extract_pose_features_kernel(const DecodeParams p, const BoneQuery q, const FeatureQuery f)
		{
			extern __shared__ __align__(16) uint8_t s_dynamic[];
			FeatureSlot* s_slot = reinterpret_cast<FeatureSlot*>(s_dynamic + q.smem_pose_offset + size_t(q.requests_per_block) * q.smem_pose_bytes);
			bone_query_block<NORM, PER_TRACK, DB>(p, q, FeatureStage<NORM, PER_TRACK, DB>{ f, s_slot });
		}

		using FeaturesKernel = void (*)(DecodeParams, BoneQuery, FeatureQuery);

		FeaturesKernel features_kernel(uint32_t normalization, bool per_track, bool database)
		{
			return with_constant<3>(normalization, [&](auto NORM) { return with_bool(per_track, [&](auto PER_TRACK) {
				return with_bool(database, [&](auto DB) -> FeaturesKernel { return extract_pose_features_kernel<NORM, PER_TRACK, DB>; }); }); });
		}
	}

	cudaError_t configure_features_kernels(int max_dynamic_smem)
	{
		cudaError_t error = cudaSuccess;
		for (uint32_t choice = 0; choice < 12 && error == cudaSuccess; ++choice)
			error = cudaFuncSetAttribute(features_kernel(choice / 4, (choice & 1) != 0, (choice & 2) != 0), cudaFuncAttributeMaxDynamicSharedMemorySize,
				max_dynamic_smem);
		return error;
	}

	// The bone query's plan with a FeatureSlot per virtual request after the pose rows
	bool plan_features_launch(const DecodeParams& params, BoneQuery& query, bool database, int max_dynamic_smem)
	{
		return plan_bones_launch(params, query, database, max_dynamic_smem, uint32_t(sizeof(FeatureSlot)));
	}

	cudaError_t launch_extract_pose_features(const DecodeParams& params, const BoneQuery& query, const FeatureQuery& features, bool database,
		cudaStream_t stream)
	{
		const uint32_t blocks = (params.num_requests + query.requests_per_block - 1) / query.requests_per_block;
		features_kernel(params.normalization, params.per_track_rounding != 0, database)<<<blocks, k_threads_per_block, query.smem_bytes, stream>>>(
			params, query, features);
		return cudaGetLastError();
	}
}
