// acl_b200/csrc/root_motion.cu -- root motion (aclb200_extract_root_motion): the root's displacement between two playback times of each
// request, across loop boundaries, composed from root samples taken with the clamp policy.
//
// A request needs up to four samples of its clip's root track: T(from), T(to) and, when playback crossed a loop boundary, the clip's two
// ends T(D) and T(0). Each sample is the root's row of aclb200_decompress_tracks for {clip, t}: the same seek (seek_request) and the bone
// decoder the bone query runs on its closure (decode_bone_row: the plain kernel's decoders, SINGLE = false), for the root only.
//
// Work decomposition, thread block = 64 requests, one lane per (request, sample slot), 8 requests per warp:
//   slot 0 from_time, slot 1 to_time, slot 2 the clamp duration D, slot 3 time 0. The lane seeks its own time and decodes the root's three
//   sub-tracks into a row in registers; the cycle end slots decode nothing when the request crosses no boundary.
//   The request's slot 0 lane gathers the other three rows with __shfl_sync, composes M (obj::compose_root_motion: rtm::qvv_inverse,
//   rtm::qvv_mul in unfused IEEE operations, object_space.cuh, shared with the pose features) and stores its 48 byte row. No pose row
//   goes through shared memory.
#include "device_common.cuh"
#include "object_space.cuh"

#include <type_traits>

namespace aclb200
{
	using namespace dev;

	namespace
	{
		constexpr uint32_t k_root_motion_slots = 4;			// from, to, the clip's end (D), its start (0)
		constexpr uint32_t k_root_motion_requests_per_block = k_threads_per_block / k_root_motion_slots;
		static_assert(32 % k_root_motion_slots == 0, "a request's slots lie in one warp");

		using obj::Qvv;
		using obj::Quat;
		using obj::Vec3;

		// the row of lane `source` of the warp, as an rtm::qvvf
		__device__ __forceinline__ Qvv<float> shuffle_row(const float4 row[3], uint32_t source)
		{
			Qvv<float> q;
			q.rotation = Quat<float>{ __shfl_sync(0xFFFFFFFFu, row[0].x, source), __shfl_sync(0xFFFFFFFFu, row[0].y, source),
				__shfl_sync(0xFFFFFFFFu, row[0].z, source), __shfl_sync(0xFFFFFFFFu, row[0].w, source) };
			q.translation = Vec3<float>{ __shfl_sync(0xFFFFFFFFu, row[1].x, source), __shfl_sync(0xFFFFFFFFu, row[1].y, source),
				__shfl_sync(0xFFFFFFFFu, row[1].z, source) };
			q.scale = Vec3<float>{ __shfl_sync(0xFFFFFFFFu, row[2].x, source), __shfl_sync(0xFFFFFFFFu, row[2].y, source),
				__shfl_sync(0xFFFFFFFFu, row[2].z, source) };
			return q;
		}

		template<int NORM, bool PER_TRACK, bool DB>
		__global__ void __launch_bounds__(k_threads_per_block)
		extract_root_motion_kernel(const DecodeParams p, const RootMotionQuery q)
		{
			using RS = typename std::conditional<DB, ReqStateDB, ReqState>::type;
			const uint32_t lane = threadIdx.x & 31u;
			const uint32_t slot = threadIdx.x & (k_root_motion_slots - 1);
			const uint64_t request_index = uint64_t(blockIdx.x) * k_root_motion_requests_per_block + threadIdx.x / k_root_motion_slots;

			// the request, its root track and whether it writes its row (an invalid clip, a root beyond the clip's tracks and too many
			// cycles leave the row as it is)
			uint32_t clip_index = 0xFFFFFFFFu;
			float from_time = 0.0f, to_time = 0.0f;
			int32_t cycles = 0;
			if (request_index < p.num_requests)
			{
				// four 4 byte loads: the ABI only promises the request array the 4 byte alignment of its fields
				const uint32_t* fields = reinterpret_cast<const uint32_t*>(q.requests + request_index);
				clip_index = __ldg(fields);
				from_time = __uint_as_float(__ldg(fields + 1));
				to_time = __uint_as_float(__ldg(fields + 2));
				cycles = int32_t(__ldg(fields + 3));
			}
			bool writes = false;
			uint32_t root = 0, clip_flags = 0;
			float duration = 0.0f;
			if (clip_index < p.num_clips)
			{
				const ClipDesc& clip = p.clips[clip_index];
				root = q.root_tracks != nullptr ? __ldg(q.root_tracks + clip_index) : 0u;
				writes = root < clip.num_tracks && cycles >= -ACLB200_MAX_ROOT_MOTION_CYCLES && cycles <= ACLB200_MAX_ROOT_MOTION_CYCLES;
				clip_flags = clip.flags;
				duration = clip.duration_clamp;
			}

			// ---- one sample per lane: seek, then the root's constant, default and animated sub-tracks into a row in registers ----
			float4 row[3] = { make_float4(0.0f, 0.0f, 0.0f, 0.0f), make_float4(0.0f, 0.0f, 0.0f, 0.0f), make_float4(0.0f, 0.0f, 0.0f, 0.0f) };
			if (writes && (slot < 2 || cycles != 0))
			{
				const float time = slot == 0 ? from_time : slot == 1 ? to_time : slot == 2 ? duration : 0.0f;
				RS rs;
				seek_request<DB>(p, aclb200_request{ clip_index, time }, uint32_t(request_index), rs);
				// the decoders write through a pointer, but at constant offsets of `row` once inlined: the row stays in registers (the kernel's
				// local memory is only the argument block of the out-of-line negative scale path, obj::qvv_mul_negative_scale)
				decode_bone_row<NORM, PER_TRACK>(p, rs, root, reinterpret_cast<uint8_t*>(row));
			}

			// ---- the request's slot 0 lane composes M from the four samples ----
			const uint32_t first = lane & ~(k_root_motion_slots - 1);
			const Qvv<float> from = shuffle_row(row, first);
			const Qvv<float> to = shuffle_row(row, first + 1);
			const Qvv<float> end = shuffle_row(row, first + 2);
			const Qvv<float> start = shuffle_row(row, first + 3);
			uint32_t flags = 0;
			if (slot == 0 && writes)
				obj::store_qvv_row(reinterpret_cast<float4*>(p.out + request_index * 48),
					obj::compose_root_motion(from, to, end, start, cycles, clip_flags, flags));
			flags = __reduce_or_sync(0xFFFFFFFFu, flags);
			if (lane == 0 && flags != 0 && q.out_flags != nullptr)
				atomicOr(q.out_flags, flags);
		}

		using RootMotionKernel = void (*)(DecodeParams, RootMotionQuery);

		RootMotionKernel root_motion_kernel(uint32_t normalization, bool per_track, bool database)
		{
			return with_constant<3>(normalization, [&](auto NORM) { return with_bool(per_track, [&](auto PER_TRACK) {
				return with_bool(database, [&](auto DB) -> RootMotionKernel { return extract_root_motion_kernel<NORM, PER_TRACK, DB>; }); }); });
		}
	}

	cudaError_t launch_extract_root_motion(const DecodeParams& params, const RootMotionQuery& query, bool database, cudaStream_t stream)
	{
		const uint32_t blocks = uint32_t((uint64_t(params.num_requests) + k_root_motion_requests_per_block - 1) / k_root_motion_requests_per_block);
		root_motion_kernel(params.normalization, params.per_track_rounding != 0, database)<<<blocks, k_threads_per_block, 0, stream>>>(params, query);
		return cudaGetLastError();
	}
}
