// acl_b200/csrc/error_metric.cu -- SURVEY 8(f1) + 8(f3): the nearest caller of the decode hot path inside ACL, on the device.
//
//   * aclb200_calculate_compression_error: acl::calculate_compression_error (includes/acl/compression/impl/track_error.impl.h:400-680
//     -> calculate_transform_track_error :225-392 / calculate_scalar_track_error :166-223) for MANY clips per call: every sample of every
//     clip is decoded by the decompress_tracks pipeline (pipeline.cu), taken to object space and measured against the raw pose with one of
//     the reference's metrics (includes/acl/compression/transform_error_metrics.h: qvvf_transform_error_metric :281-385,
//     qvvf_matrix3x4f_transform_error_metric :389-464, additive_qvvf_transform_error_metric<format> :470-526 with its additive base);
//     one {index, error, sample_time} per clip comes back, the poses never leave the GPU.
//   * aclb200_decompress_all_samples: the sampling loop of that measurement and of acl::convert_track_list (impl/convert.impl.h:146-232)
//     as an entry point of its own.
//   * aclb200_local_to_object_space: qvvf_transform_error_metric::local_to_object_space (transform_error_metrics.h:289-310) as a pose
//     consumer of its own (the hierarchy walk a skinning / blending stage starts with).
//
// Work decomposition: ONE WARP PER POSE. The reference walks a pose bone by bone because a bone needs its parent's object transform; here
// the warp takes 32 consecutive bones at a time and resolves them in wavefronts (object_space.cuh, shared with the object space decode of
// kernels.cu). Object transforms live in shared memory as [component][bone] planes so that 32 lanes reading 32
// different parents hit 32 different banks; a bone's local transform is parked in the slot its object transform will take. The
// measurement itself (three shell points through both transforms) runs after the chunk's wavefronts with every lane busy, and the raw and
// the lossy pose travel together as f32x2 pairs (one scalar operation per lane on sm_90).
//
// Every float operation is the reference's, in its order, never fused (the library is built with --fmad=false and uses the _rn
// intrinsics). The one exception is rtm::quat_normalize, whose SSE2 code starts from the CPU specific rsqrtss estimate
// (external/rtm/includes/rtm/quatf.h:917-953) and cannot be reproduced bit for bit by anyone: the IEEE 1 / sqrt stands in for it (the
// tests' CPU restatement has both flavours; errors agree with the reference within 5e-5 on poses tens of units across,
// tests/test_gpu_error_metric.py). The matrix metric never normalises: it is bit-identical to the reference itself.
#include "context.h"
#include "object_space.cuh"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <type_traits>
#include <vector>

namespace aclb200
{
	namespace
	{
		using namespace obj;

		// One clip to measure, in processing order (a chunk = a run of jobs whose poses fit the scratch).
		struct alignas(16) ErrorJobDev
		{
			uint32_t clip;
			uint32_t num_samples;
			uint32_t num_tracks;
			uint32_t skeleton_offset;
			float    sample_rate;
			float    duration;
			uint32_t chunk_first_pose;		// first pose of the job inside the chunk's scratch
			uint32_t job_index;				// slot of the result (the caller's job order)
			uint64_t first_raw_pose;
			uint64_t out_pose_base;			// first row of the job in the optional per bone error matrix
			uint64_t first_base_pose;		// additive base: pose index of sample 0 in the base poses
			uint32_t additive_format;		// acl::additive_clip_format8 (0 = the clip is not additive)
			uint32_t pad;
		};
		static_assert(sizeof(ErrorJobDev) == 64, "ErrorJobDev is 64 bytes");

		struct ErrorParams
		{
			const ErrorJobDev* jobs;		// the chunk's jobs
			uint32_t num_jobs;
			uint32_t num_poses;				// of the chunk
			aclb200_request* requests;		// [num_poses] (setup kernel output)
			uint32_t* pose_jobs;			// [num_poses] index into `jobs`
			const uint8_t* raw_poses;
			const uint8_t* lossy_poses;		// chunk scratch, pose p at p * pose_stride
			const uint8_t* base_poses;		// additive base poses, or nullptr
			uint64_t pose_stride;
			const uint32_t* parent_indices;
			const float* shell_distances;
			const uint32_t* output_indices;	// or nullptr
			unsigned long long* keys;		// [all jobs] arg max accumulators
			uint32_t* flags;				// [all jobs]
			float* error_matrix;			// or nullptr
			uint32_t error_stride;			// floats per row of the matrix
			uint32_t plane_stride;			// floats per [component] plane of a warp's object transforms
			uint32_t components;			// scalar clips
		};

		// rtm::qvv_mul_point3(shell point, qvv) (qvvf.h:370-373) for the three shell points of construct_sphere_shell
		// (transform_error_metrics.h:261-266): (d, 0, 0), (0, d, 0), (0, 0, d). quat_mul_vector3 of a vector with two zero components: the
		// terms that multiply a zero are dropped. They contribute +-0 to sums, which changes nothing but the sign of a sum that is itself
		// zero, and the distance squares every difference: for finite transforms the measured error is bit-identical to the full sequence
		// (a non-finite transform gives NaN there -- 0 * inf -- and may not here).
		template<class V>
		__device__ __forceinline__ void shell_points(const Fp<V>& fp, const Qvv<V>& q, float shell_distance, Vec3<V> out[3])
		{
			const Quat<V>& r = q.rotation;
			const V d = fp.splat(shell_distance);
			{
				const V a = fp.mul(q.scale.x, d);
				const V t0 = fp.mul(a, r.w), t1 = fp.mul(a, r.z), u2 = fp.mul(a, r.y), t3 = fp.mul(a, r.x);		// t2 = -u2
				out[0].x = fp.add(fp.sub(fp.add(fp.mul(r.w, t0), fp.mul(r.x, t3)), fp.add(fp.mul(r.y, u2), fp.mul(r.z, t1))), q.translation.x);
				out[0].y = fp.add(fp.add(fp.add(fp.mul(r.w, t1), fp.mul(r.x, u2)), fp.add(fp.mul(r.y, t3), fp.mul(r.z, t0))), q.translation.y);
				out[0].z = fp.add(fp.add(fp.sub(fp.mul(r.x, t1), fp.mul(r.w, u2)), fp.sub(fp.mul(r.z, t3), fp.mul(r.y, t0))), q.translation.z);
			}
			{
				const V b = fp.mul(q.scale.y, d);
				const V u0 = fp.mul(b, r.z), t1 = fp.mul(b, r.w), t2 = fp.mul(b, r.x), t3 = fp.mul(b, r.y);		// t0 = -u0
				out[1].x = fp.add(fp.add(fp.sub(fp.mul(r.x, t3), fp.mul(r.w, u0)), fp.sub(fp.mul(r.y, t2), fp.mul(r.z, t1))), q.translation.x);
				out[1].y = fp.add(fp.add(fp.sub(fp.mul(r.w, t1), fp.mul(r.x, t2)), fp.sub(fp.mul(r.y, t3), fp.mul(r.z, u0))), q.translation.y);
				out[1].z = fp.add(fp.add(fp.add(fp.mul(r.w, t2), fp.mul(r.x, t1)), fp.add(fp.mul(r.z, t3), fp.mul(r.y, u0))), q.translation.z);
			}
			{
				const V c = fp.mul(q.scale.z, d);
				const V t0 = fp.mul(c, r.y), u1 = fp.mul(c, r.x), t2 = fp.mul(c, r.w), t3 = fp.mul(c, r.z);		// t1 = -u1
				out[2].x = fp.add(fp.add(fp.add(fp.mul(r.w, t0), fp.mul(r.x, t3)), fp.add(fp.mul(r.y, t2), fp.mul(r.z, u1))), q.translation.x);
				out[2].y = fp.add(fp.sub(fp.add(fp.mul(r.y, t3), fp.mul(r.z, t0)), fp.add(fp.mul(r.w, u1), fp.mul(r.x, t2))), q.translation.y);
				out[2].z = fp.add(fp.add(fp.sub(fp.mul(r.w, t2), fp.mul(r.x, u1)), fp.sub(fp.mul(r.z, t3), fp.mul(r.y, t0))), q.translation.z);
			}
		}

		__device__ __forceinline__ float max_ss(float a, float b) { return a > b ? a : b; }		// _mm_max_ss: the second operand when unordered

		// qvvf_transform_error_metric::calculate_error, transform_error_metrics.h:335-358: per shell point
		// rtm::vector_distance3_as_scalar(raw, lossy) (vector4f.h:2260-2264: dot3 = (x2 + y2) + z2, :1899-1906; sqrtss), then the largest
		__device__ __forceinline__ float calculate_error(const Fp<float2>& fp, const Qvv<float2>& object, float shell_distance)
		{
			Vec3<float2> points[3];
			shell_points(fp, object, shell_distance, points);
			float error = 0.0f;
			#pragma unroll
			for (int axis = 0; axis < 3; ++axis)
			{
				const float dx = __fsub_rn(points[axis].x.x, points[axis].x.y);
				const float dy = __fsub_rn(points[axis].y.x, points[axis].y.y);
				const float dz = __fsub_rn(points[axis].z.x, points[axis].z.y);
				const float axis_error = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
				error = axis == 0 ? axis_error : max_ss(error, axis_error);
			}
			return error;
		}

		// calculate_error of the matrix metric (:438-463): rtm::matrix_mul_point3 (matrix3x4f.h:326-336) of the shell points (d, 0, 0), (0, d, 0),
		// (0, 0, d) comes down to d * axis + w_axis once the terms that multiply a zero component are dropped (same argument as shell_points)
		__device__ __forceinline__ float matrix_calculate_error(const Fp<float2>& fp, const Mat34<float2>& object, float shell_distance)
		{
			const float2 d = fp.splat(shell_distance);
			float error = 0.0f;
			#pragma unroll
			for (int axis = 0; axis < 3; ++axis)
			{
				const float2 x = fp.add(fp.mul(d, object.m[axis][0]), object.m[3][0]);
				const float2 y = fp.add(fp.mul(d, object.m[axis][1]), object.m[3][1]);
				const float2 z = fp.add(fp.mul(d, object.m[axis][2]), object.m[3][2]);
				const float dx = __fsub_rn(x.x, x.y), dy = __fsub_rn(y.x, y.y), dz = __fsub_rn(z.x, z.y);
				const float axis_error = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
				error = axis == 0 ? axis_error : max_ss(error, axis_error);
			}
			return error;
		}

		struct Bone48 { float4 rotation, translation, scale; };

		__device__ __forceinline__ Bone48 load_bone48(const uint8_t* bone)
		{
			Bone48 out;
			out.rotation = __ldg(reinterpret_cast<const float4*>(bone));
			out.translation = __ldg(reinterpret_cast<const float4*>(bone + 16));
			out.scale = __ldg(reinterpret_cast<const float4*>(bone + 32));
			return out;
		}

		__device__ __forceinline__ Qvv<float> make_qvv(const Bone48& a)
		{
			Qvv<float> q;
			q.rotation = Quat<float>{ a.rotation.x, a.rotation.y, a.rotation.z, a.rotation.w };
			q.translation = Vec3<float>{ a.translation.x, a.translation.y, a.translation.z };
			q.scale = Vec3<float>{ a.scale.x, a.scale.y, a.scale.z };
			return q;
		}

		__device__ __forceinline__ Qvv<float2> make_qvv(const Bone48& a, const Bone48& b)
		{
			Qvv<float2> q;
			q.rotation = Quat<float2>{ make_float2(a.rotation.x, b.rotation.x), make_float2(a.rotation.y, b.rotation.y), make_float2(a.rotation.z, b.rotation.z), make_float2(a.rotation.w, b.rotation.w) };
			q.translation = Vec3<float2>{ make_float2(a.translation.x, b.translation.x), make_float2(a.translation.y, b.translation.y), make_float2(a.translation.z, b.translation.z) };
			q.scale = Vec3<float2>{ make_float2(a.scale.x, b.scale.x), make_float2(a.scale.y, b.scale.y), make_float2(a.scale.z, b.scale.z) };
			return q;
		}

		template<class V> __device__ __forceinline__ Qvv<V> make_qvv_pair(const Qvv<float>& q);
		template<> __device__ __forceinline__ Qvv<float> make_qvv_pair<float>(const Qvv<float>& q) { return q; }
		template<> __device__ __forceinline__ Qvv<float2> make_qvv_pair<float2>(const Qvv<float>& q)
		{
			Qvv<float2> out;
			out.rotation = Quat<float2>{ make_float2(q.rotation.x, q.rotation.x), make_float2(q.rotation.y, q.rotation.y), make_float2(q.rotation.z, q.rotation.z), make_float2(q.rotation.w, q.rotation.w) };
			out.translation = Vec3<float2>{ make_float2(q.translation.x, q.translation.x), make_float2(q.translation.y, q.translation.y), make_float2(q.translation.z, q.translation.z) };
			out.scale = Vec3<float2>{ make_float2(q.scale.x, q.scale.x), make_float2(q.scale.y, q.scale.y), make_float2(q.scale.z, q.scale.z) };
			return out;
		}

		// planes[bone] = qvv_mul(planes[bone] (the additive transform), base): the `relative` additive format, every stream
		template<class V>
		__device__ __noinline__ void apply_relative_slow(V* planes, uint32_t plane_stride, uint32_t bone, const Qvv<float>* base)
		{
			for (int stream = 0; stream < Streams<V>::count; ++stream)
				write_stream(planes, plane_stride, bone, stream, qvv_mul_any(read_stream(planes, plane_stride, bone, stream), *base));
		}

		// arg max key: larger error wins, then the EARLIER (sample, bone) -- the reference keeps the first maximum it meets walking samples
		// then bones with a strict `>` (track_error.impl.h:367-372). Errors are >= +0 or NaN (never kept), so their bit patterns order like
		// the values. 0 = nothing measured yet.
		__device__ __forceinline__ unsigned long long error_key(float error, uint32_t linear_index)
		{
			return ((static_cast<unsigned long long>(__float_as_uint(error)) + 1ull) << 32) | static_cast<unsigned long long>(~linear_index);
		}

		// sample_time = rtm::scalar_min(float(sample_index) / sample_rate, duration), track_error.impl.h:337 / :189
		__device__ __forceinline__ float error_sample_time(uint32_t sample, float sample_rate, float duration)
		{
			const float t = __fdiv_rn(static_cast<float>(sample), sample_rate);
			return t < duration ? t : duration;
		}

		// One thread per pose of the chunk: which job it belongs to, and the (clip, sample_time) request the decode kernels take.
		__global__ void build_error_requests_kernel(ErrorParams p)
		{
			const uint32_t pose = blockIdx.x * blockDim.x + threadIdx.x;
			if (pose >= p.num_poses)
				return;
			uint32_t lo = 0, hi = p.num_jobs;			// last job whose first pose is <= pose (jobs without samples share a first pose: skipped)
			while (hi - lo > 1)
			{
				const uint32_t mid = (lo + hi) >> 1;
				if (p.jobs[mid].chunk_first_pose <= pose)
					lo = mid;
				else
					hi = mid;
			}
			const ErrorJobDev job = p.jobs[lo];
			aclb200_request request;
			request.clip = job.clip;
			request.sample_time = error_sample_time(pose - job.chunk_first_pose, job.sample_rate, job.duration);
			p.requests[pose] = request;
			p.pose_jobs[pose] = lo;
		}

		// MODE 0: error measurement (two pose streams: raw + lossy), MODE 1: local_to_object_space of one stream, object poses written out.
		struct ObjectSpaceParams
		{
			const uint8_t* local_poses;
			uint8_t* object_poses;
			uint64_t num_poses;
			uint64_t pose_stride;
			uint32_t num_tracks;
			const uint32_t* parent_indices;
			uint32_t plane_stride;
			uint32_t* flags;				// [1]
		};

		// METRIC (MODE 0 only): 0 = qvvf_transform_error_metric, 1 = qvvf_matrix3x4f_transform_error_metric
		template<int MODE, int METRIC = 0>
		__global__ void __launch_bounds__(256, 2) object_space_kernel(ErrorParams ep, ObjectSpaceParams op)
		{
			using V = typename std::conditional<MODE == 0, float2, float>::type;
			extern __shared__ __align__(16) uint8_t object_plane_bytes[];
			const uint32_t lane = threadIdx.x & 31u;
			const uint32_t warp = threadIdx.x >> 5;
			const uint32_t warps_per_block = blockDim.x >> 5;
			const uint32_t plane_stride = MODE == 0 ? ep.plane_stride : op.plane_stride;
			constexpr uint32_t k_components = METRIC == 1 ? 12u : k_object_components;
			V* planes = reinterpret_cast<V*>(object_plane_bytes) + size_t(warp) * k_components * plane_stride;
			const uint64_t num_poses = MODE == 0 ? uint64_t(ep.num_poses) : op.num_poses;
			const Fp<V> fp{};

			for (uint64_t pose = uint64_t(blockIdx.x) * warps_per_block + warp; pose < num_poses; pose += uint64_t(gridDim.x) * warps_per_block)
			{
				uint32_t num_tracks, sample = 0, job_slot = 0;
				const uint8_t* raw_pose;
				const uint8_t* lossy_pose = nullptr;
				const uint32_t* parents;
				const float* shells = nullptr;
				const uint32_t* output_indices = nullptr;
				float* error_row = nullptr;
				const uint8_t* base_pose = nullptr;
				uint32_t additive_format = 0;
				if (MODE == 0)
				{
					const ErrorJobDev job = ep.jobs[ep.pose_jobs[pose]];
					if (ep.base_poses != nullptr && job.additive_format != 0)
					{
						additive_format = job.additive_format;
						base_pose = ep.base_poses + (job.first_base_pose + (uint32_t(pose) - job.chunk_first_pose)) * ep.pose_stride;
					}
					num_tracks = job.num_tracks;
					sample = uint32_t(pose) - job.chunk_first_pose;
					job_slot = job.job_index;
					raw_pose = ep.raw_poses + (job.first_raw_pose + sample) * ep.pose_stride;
					lossy_pose = ep.lossy_poses + pose * ep.pose_stride;
					parents = ep.parent_indices + job.skeleton_offset;
					shells = ep.shell_distances + job.skeleton_offset;
					output_indices = ep.output_indices != nullptr ? ep.output_indices + job.skeleton_offset : nullptr;
					if (ep.error_matrix != nullptr)
						error_row = ep.error_matrix + (job.out_pose_base + sample) * ep.error_stride;
				}
				else
				{
					num_tracks = op.num_tracks;
					raw_pose = op.local_poses + pose * op.pose_stride;
					parents = op.parent_indices;
				}

				float best_error = -1.0f;				// track_error.impl.h:333
				uint32_t best_bone = k_invalid_track;
				uint32_t pose_flags = 0;

				for (uint32_t base = 0; base < num_tracks; base += 32)
				{
					const uint32_t bone = base + lane;
					const bool active = bone < num_tracks;
					// Lanes past the last bone load the last bone again (their results are never stored): no value of the loop below depends
					// on a branch, which keeps the packed pairs in aligned register pairs from the load to the arithmetic.
					const uint32_t load_bone = active ? bone : num_tracks - 1;
					uint32_t parent = __ldg(parents + load_bone);
					const Bone48 raw_local = load_bone48(raw_pose + size_t(load_bone) * 48);
					float shell = 0.0f;
					Qvv<V> local;						// the bone's local transform (MODE 0: raw and lossy as one packed value)
					if constexpr (MODE == 0)
					{
						shell = __ldg(shells + load_bone);
						// remap_output (track_error.impl.h:522-532): the raw value stands in for a bone the compressed clip does not output
						const uint32_t output_index = output_indices != nullptr ? __ldg(output_indices + load_bone) : load_bone;
						const uint8_t* lossy_bone = output_index != k_invalid_track ? lossy_pose + size_t(output_index) * 48 : raw_pose + size_t(load_bone) * 48;
						local = make_qvv(raw_local, load_bone48(lossy_bone));
					}
					else
						local = make_qvv(raw_local);
					if (parent_follows(active, bone, parent))
					{
						pose_flags |= ACLB200_ERROR_FLAG_INVALID_SKELETON;
						parent = k_invalid_track;
					}

					// The local transform is parked in the bone's own slot of the planes: the object transform will overwrite it. Nothing
					// packed lives in registers across a branch (see the out of line paths above); a root is done at this point (:300-301).
					if (active)
					{
						if constexpr (METRIC == 1)
							store_matrix_planes(planes, plane_stride, bone, matrix_from_qvv(fp, local));		// convert_transforms
						else
							store_planes(planes, plane_stride, bone, local);
					}
					if (MODE == 0 && METRIC == 0 && additive_format != 0 && active)
					{
						// apply_additive_to_base on the raw and on the lossy pose before the walk (track_error.impl.h:358-359)
						const Qvv<float> base = make_qvv(load_bone48(base_pose + size_t(bone) * 48));
						const Qvv<V> base_pair = make_qvv_pair<V>(base);
						if (additive_format == 1 && takes_negative_branch(fp, local.scale, base_pair.scale))
						{
							pose_flags |= ACLB200_ERROR_FLAG_NEGATIVE_SCALE;
							apply_relative_slow(planes, plane_stride, bone, &base);
						}
						else
							store_planes(planes, plane_stride, bone, apply_additive_to_base_positive(fp, additive_format, base_pair, local));
					}
					__syncwarp();

					// the hierarchy walk of the chunk, in wavefronts: a lane computes once its parent's object transform is in shared memory
					wavefront_walk(active, parent, base, [&]()
					{
						if constexpr (METRIC == 1)
							store_matrix_planes(planes, plane_stride, bone, matrix_mul(fp, load_matrix_planes(planes, plane_stride, bone), load_matrix_planes(planes, plane_stride, parent)));
						else
						{
							const Qvv<V> mine = load_planes(planes, plane_stride, bone);
							const Qvv<V> above = load_planes(planes, plane_stride, parent);
							if (takes_negative_branch(fp, mine.scale, above.scale))
							{
								pose_flags |= ACLB200_ERROR_FLAG_NEGATIVE_SCALE;
								object_transform_slow(planes, plane_stride, bone, parent);
							}
							else
							{
								// rtm::qvv_normalize(rtm::qvv_mul(local, parent_object)), qvvf.h:426-430
								Qvv<V> object = qvv_mul_positive(fp, mine, above);
								object.rotation = quat_normalize(fp, object.rotation);
								store_planes(planes, plane_stride, bone, object);
							}
						}
					});

					// every lane of the chunk at once: the measurement (or the store) needs nothing but the lane's own object transform
					if (active)
					{
						if constexpr (MODE == 0)
						{
							float error;
							if constexpr (METRIC == 1)
								error = matrix_calculate_error(fp, load_matrix_planes(planes, plane_stride, bone), shell);
							else
								error = calculate_error(fp, load_planes(planes, plane_stride, bone), shell);
							if (error_row != nullptr)
								error_row[bone] = error;
							if (error > best_error)
							{
								best_error = error;
								best_bone = bone;
							}
						}
						else
						{
							const Qvv<V> object = load_planes(planes, plane_stride, bone);
							float4* out = reinterpret_cast<float4*>(op.object_poses + pose * op.pose_stride + size_t(bone) * 48);
							out[0] = make_float4(object.rotation.x, object.rotation.y, object.rotation.z, object.rotation.w);
							out[1] = make_float4(object.translation.x, object.translation.y, object.translation.z, 0.0f);
							out[2] = make_float4(object.scale.x, object.scale.y, object.scale.z, 0.0f);
						}
					}
				}
				__syncwarp();		// the next pose overwrites the planes

				if (MODE == 0)
				{
					// first maximum of the pose: larger error, then the smaller bone index (a lane's own bones already come in rising order)
					#pragma unroll
					for (int offset = 16; offset > 0; offset >>= 1)
					{
						const float other_error = __shfl_xor_sync(0xFFFFFFFFu, best_error, offset);
						const uint32_t other_bone = __shfl_xor_sync(0xFFFFFFFFu, best_bone, offset);
						if (other_error > best_error || (other_error == best_error && other_bone < best_bone))
						{
							best_error = other_error;
							best_bone = other_bone;
						}
					}
					pose_flags = __reduce_or_sync(0xFFFFFFFFu, pose_flags);
					if (lane == 0)
					{
						if (best_bone != k_invalid_track)
							atomicMax(ep.keys + job_slot, error_key(best_error, sample * num_tracks + best_bone));
						if (pose_flags != 0)
							atomicOr(ep.flags + job_slot, pose_flags);
					}
				}
				else
				{
					pose_flags = __reduce_or_sync(0xFFFFFFFFu, pose_flags);
					if (lane == 0 && pose_flags != 0 && op.flags != nullptr)
						atomicOr(op.flags, pose_flags);
				}
			}
		}

		// calculate_scalar_track_error (track_error.impl.h:166-223) + get_scalar_track_error (:51-101): one thread per (pose, track)
		__global__ void scalar_error_kernel(ErrorParams p, uint32_t max_tracks)
		{
			const uint64_t item = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
			const uint64_t pose = item / max_tracks;
			const uint32_t track = uint32_t(item % max_tracks);
			if (pose >= p.num_poses)
				return;
			const ErrorJobDev job = p.jobs[p.pose_jobs[pose]];
			if (track >= job.num_tracks)
				return;
			const uint32_t sample = uint32_t(pose) - job.chunk_first_pose;
			const float* raw = reinterpret_cast<const float*>(p.raw_poses + (job.first_raw_pose + sample) * p.pose_stride) + size_t(track) * p.components;
			const float* lossy = reinterpret_cast<const float*>(p.lossy_poses + pose * p.pose_stride) + size_t(track) * p.components;
			float e[4] = { 0.0f, 0.0f, 0.0f, 0.0f };
			for (uint32_t c = 0; c < p.components; ++c)
				e[c] = fabsf(__fsub_rn(__ldg(raw + c), __ldg(lossy + c)));
			// vector_get_max_component (external/rtm/includes/rtm/impl/vector_common.h:508-523): max(max(x, z), max(y, w)); float1f broadcasts x
			const float error = p.components == 1 ? e[0] : max_ss(max_ss(e[0], e[2]), max_ss(e[1], e[3]));
			if (p.error_matrix != nullptr)
				p.error_matrix[(job.out_pose_base + sample) * p.error_stride + track] = error;
			if (error >= 0.0f)			// never a NaN: `error > result.error` is false for it
				atomicMax(p.keys + job.job_index, error_key(error, sample * job.num_tracks + track));
		}

		// One thread per job: the arg max key back into acl::track_error
		__global__ void finalize_error_kernel(const ErrorJobDev* jobs, uint32_t num_jobs, const unsigned long long* keys, const uint32_t* flags, aclb200_track_error* out)
		{
			const uint32_t index = blockIdx.x * blockDim.x + threadIdx.x;
			if (index >= num_jobs)
				return;
			const ErrorJobDev job = jobs[index];
			aclb200_track_error result;
			result.index = k_invalid_track;			// track_error(), compression/track_error.h:48-62
			result.error = 0.0f;
			result.sample_time = 0.0f;
			result.flags = flags[job.job_index];
			if (job.num_samples != 0 && job.num_tracks != 0)
			{
				const unsigned long long key = keys[job.job_index];
				if (key == 0)
					result.error = -1.0f;				// nothing compared greater than -1: every error was a NaN
				else
				{
					const uint32_t linear = ~uint32_t(key & 0xFFFFFFFFull);
					const uint32_t sample = linear / job.num_tracks;
					result.index = linear - sample * job.num_tracks;
					result.error = __uint_as_float(uint32_t(key >> 32) - 1u);
					result.sample_time = error_sample_time(sample, job.sample_rate, job.duration);
				}
			}
			out[job.job_index] = result;
		}

		uint32_t plane_stride_for(uint32_t num_tracks)
		{
			return (std::max(num_tracks, 1u) + 31u) & ~31u;
		}

		// warps per block so that the object transform planes fit; 0 = the skeleton is too wide for shared memory
		uint32_t warps_for(uint32_t plane_stride, uint32_t floats_per_bone, int max_dynamic_smem)
		{
			const size_t per_warp = size_t(floats_per_bone) * plane_stride * sizeof(float);
			const size_t budget = max_dynamic_smem > 0 ? size_t(max_dynamic_smem) : 0;
			if (per_warp > budget)
				return 0;
			// two blocks per SM when they fit (the wavefront loop leaves lanes idle: more warps hide it)
			const size_t block_budget = std::max(per_warp, std::min(budget, size_t(100) * 1024));
			return uint32_t(std::min<size_t>(8, block_budget / per_warp));
		}

		// The context's scratch is shared by every call, whatever its stream: a call makes its stream wait for the previous user's last
		// reader before it writes (error_scratch_done), and records the event after its own last reader (ScratchUse).
		aclb200_status grow_scratch(aclb200_context* context, size_t bytes)
		{
			if (context->error_scratch_done == nullptr)
			{
				const cudaError_t error = cudaEventCreateWithFlags(&context->error_scratch_done, cudaEventDisableTiming);
				if (error != cudaSuccess)
				{
					context->error_scratch_done = nullptr;
					return check_cuda(context, error, "error scratch: event creation");
				}
			}
			if (context->error_scratch_bytes >= bytes)
				return ACLB200_OK;
			// the old buffer may still be read by a call on another stream
			cudaError_t error = cudaEventSynchronize(context->error_scratch_done);
			if (error != cudaSuccess)
				return check_cuda(context, error, "error scratch: waiting for its last reader");
			cudaFree(context->d_error_scratch);
			context->d_error_scratch = nullptr;
			context->error_scratch_bytes = 0;
			error = cudaMalloc(&context->d_error_scratch, bytes);
			if (error != cudaSuccess)
				return check_cuda(context, error, "calculate_compression_error: scratch allocation");
			context->error_scratch_bytes = bytes;
			return ACLB200_OK;
		}

		// From the stream's wait to the end of the call: every return records the scratch's last use on the call's stream, after whatever
		// it enqueued.
		struct ScratchUse
		{
			aclb200_context* context;
			cudaStream_t stream;
			cudaError_t wait() const { return cudaStreamWaitEvent(stream, context->error_scratch_done, 0); }
			~ScratchUse() { cudaEventRecord(context->error_scratch_done, stream); }
		};

		size_t align_up(size_t value, size_t alignment) { return (value + alignment - 1) / alignment * alignment; }
	}

	cudaError_t configure_error_kernels(int optin_limit)
	{
		cudaError_t error = cudaFuncSetAttribute(object_space_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin_limit);
		if (error == cudaSuccess)
			error = cudaFuncSetAttribute(object_space_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin_limit);
		if (error == cudaSuccess)
			error = cudaFuncSetAttribute(object_space_kernel<0, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin_limit);
		return error;
	}
}

using namespace aclb200;

extern "C"
{
	aclb200_status aclb200_local_to_object_space(aclb200_context* context, const void* d_local_poses, void* d_object_poses, uint64_t num_poses,
		uint32_t num_tracks, uint64_t pose_stride_bytes, const uint32_t* d_parent_indices, uint32_t* d_out_flags, void* stream)
	{
		if (context == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		if (num_poses == 0 || num_tracks == 0)
			return ACLB200_OK;
		if (d_local_poses == nullptr || d_object_poses == nullptr || d_parent_indices == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "local_to_object_space: null pose / parent pointer");
		uint64_t stride = pose_stride_bytes;
		aclb200_status status = check_qvvf_rows(context, { d_local_poses, d_object_poses }, num_tracks, stride, "local_to_object_space");
		if (status != ACLB200_OK)
			return status;

		ObjectSpaceParams op = {};
		op.local_poses = static_cast<const uint8_t*>(d_local_poses);
		op.object_poses = static_cast<uint8_t*>(d_object_poses);
		op.num_poses = num_poses;
		op.pose_stride = stride;
		op.num_tracks = num_tracks;
		op.parent_indices = d_parent_indices;
		op.plane_stride = plane_stride_for(num_tracks);
		op.flags = d_out_flags;
		const uint32_t warps = warps_for(op.plane_stride, k_object_components, context->max_dynamic_smem);
		if (warps == 0)
			return set_error(context, ACLB200_ERR_UNSUPPORTED, "local_to_object_space: the skeleton's object transforms do not fit in shared memory");

		cudaSetDevice(context->device);
		cudaStream_t cuda_stream = static_cast<cudaStream_t>(stream);
		status = clear_out_flags(context, d_out_flags, cuda_stream, "local_to_object_space");
		if (status != ACLB200_OK)
			return status;
		const uint64_t blocks_needed = (num_poses + warps - 1) / warps;
		const uint32_t blocks = uint32_t(std::min<uint64_t>(blocks_needed, uint64_t(context->num_sms) * 32));
		const size_t smem = size_t(warps) * k_object_components * op.plane_stride * sizeof(float);
		object_space_kernel<1><<<blocks, warps * 32, smem, cuda_stream>>>(ErrorParams{}, op);
		const cudaError_t error = cudaGetLastError();
		if (error == cudaSuccess)
			context->launch_count++;
		return check_cuda(context, error, "local_to_object_space");
	}

	static aclb200_status calculate_compression_error_impl(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_error_job* jobs,
		uint32_t num_jobs, const void* d_raw_poses, const uint32_t* d_parent_indices, const float* d_shell_distances,
		const uint32_t* d_output_indices, const void* d_base_poses, const aclb200_options* options, aclb200_track_error* d_out_errors,
		float* d_out_error_matrix, void* stream)
	{
		if (context == nullptr || clipset == nullptr || options == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "null context / clipset / options");
		if (options->struct_size != sizeof(aclb200_options))
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "options.struct_size does not match this library, call aclb200_default_options()");
		if (num_jobs == 0)
			return ACLB200_OK;
		if (jobs == nullptr || d_raw_poses == nullptr || d_out_errors == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "calculate_compression_error: null jobs / raw poses / output");
		const bool is_transform = clipset->info.track_type == ACLB200_TRACK_QVVF;
		if (is_transform && (d_parent_indices == nullptr || d_shell_distances == nullptr))
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "calculate_compression_error: transform clips need parent indices and shell distances");
		// The reference measures with a debug_track_writer that skips default sub-tracks over a buffer holding the bind pose
		// (track_error.impl.h:497-501, debug_track_writer.h:75-101): here the bind pose arrives as constant / variable defaults.
		if (is_transform && (options->default_rotation_mode == ACLB200_DEFAULT_SKIPPED || options->default_translation_mode == ACLB200_DEFAULT_SKIPPED
			|| options->default_scale_mode == ACLB200_DEFAULT_SKIPPED || (options->skip_mask & 7u) != 0 || options->d_skip_track_mask != nullptr))
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "calculate_compression_error: skipped sub-tracks have no value to measure, pass the bind pose as constant / variable defaults");
		if (options->rounding_policy == ACLB200_ROUND_PER_TRACK || options->d_request_policies != nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "calculate_compression_error picks the rounding policy itself (nearest, none for stripped clips)");

		const uint32_t components = is_transform ? 0u : (clipset->info.track_type <= 3 ? clipset->info.track_type + 1 : 4u);
		const uint32_t bone_stride = is_transform ? 48u : components * 4u;
		const uint64_t stride = options->pose_stride_bytes != 0 ? options->pose_stride_bytes : uint64_t(clipset->info.max_tracks) * bone_stride;
		const uint64_t alignment = is_transform ? 16 : 4;
		if ((stride % alignment) != 0 || (reinterpret_cast<uintptr_t>(d_raw_poses) % alignment) != 0 || (reinterpret_cast<uintptr_t>(d_base_poses) % alignment) != 0)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "calculate_compression_error: raw poses must be 16 byte aligned rtm::qvvf rows (4 byte aligned scalar rows)");

		// jobs in processing order: the clips sought with `nearest`, then the ones sought with `none` (stripped key frames leave holes
		// nearest would land in, track_error.impl.h:556-559); each group is decoded by launches of its own
		std::vector<ErrorJobDev> ordered;
		ordered.reserve(num_jobs);
		std::vector<uint64_t> out_base(num_jobs);
		uint64_t total_poses = 0;
		uint32_t widest = 0;
		for (uint32_t index = 0; index < num_jobs; ++index)
		{
			const aclb200_error_job& job = jobs[index];
			if (job.clip >= clipset->info.num_clips)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "calculate_compression_error: job names a clip outside the clip set");
			if (uint64_t(job.num_tracks) * bone_stride > stride)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "calculate_compression_error: job has more tracks than a pose row holds");
			if (d_output_indices == nullptr && job.num_tracks != clipset->host_clips[job.clip].num_tracks)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "calculate_compression_error: raw and compressed track counts differ (pass output indices)");
			if (job.error_metric > ACLB200_METRIC_QVVF_MATRIX3X4F || (job.error_metric != ACLB200_METRIC_QVVF && job.additive_format != 0))
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "calculate_compression_error: unknown error metric, or the matrix metric with an additive base (the reference does not implement that either)");
			if (job.additive_format > 3 || (job.additive_format != 0 && (d_base_poses == nullptr || !is_transform)))
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "calculate_compression_error: additive format out of range, or an additive job without base poses");
			if (uint64_t(job.num_samples) * std::max(job.num_tracks, 1u) > 0xFFFFFFFFull)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "calculate_compression_error: samples x tracks of a job must fit 32 bits");
			out_base[index] = total_poses;
			total_poses += job.num_samples;
			widest = std::max(widest, job.num_tracks);
		}
		// groups: (rounding policy) x (error metric): each is decoded and measured by launches of its own
		size_t group_begin[5] = { 0, 0, 0, 0, 0 };
		for (uint32_t pass = 0; pass < 4; ++pass)
		{
			for (uint32_t index = 0; index < num_jobs; ++index)
			{
				const aclb200_error_job& job = jobs[index];
				const bool stripped = (clipset->host_clips[job.clip].flags & k_clip_stripped) != 0;
				if (stripped != ((pass >> 1) == 1) || (is_transform ? job.error_metric : 0u) != (pass & 1u))
					continue;
				ErrorJobDev dev = {};
				dev.clip = job.clip;
				dev.num_samples = job.num_samples;
				dev.num_tracks = job.num_tracks;
				dev.skeleton_offset = job.skeleton_offset;
				dev.sample_rate = job.sample_rate;
				dev.duration = job.duration;
				dev.job_index = index;
				dev.first_raw_pose = job.first_raw_pose;
				dev.first_base_pose = job.first_base_pose;
				dev.additive_format = job.additive_format;
				dev.out_pose_base = out_base[index];
				ordered.push_back(dev);
			}
			group_begin[pass + 1] = ordered.size();
		}

		const uint32_t plane_stride = plane_stride_for(widest);
		const uint32_t warps_by_metric[2] = { is_transform ? warps_for(plane_stride, 2 * k_object_components, context->max_dynamic_smem) : 8u,
			is_transform ? warps_for(plane_stride, 2 * 12, context->max_dynamic_smem) : 8u };
		for (uint32_t metric = 0; metric < 2; ++metric)
		{
			// groups are ordered (nearest, metric 0), (nearest, metric 1), (none, metric 0), (none, metric 1)
			const size_t jobs_of_metric = (group_begin[metric + 1] - group_begin[metric]) + (group_begin[metric + 3] - group_begin[metric + 2]);
			if (warps_by_metric[metric] == 0 && jobs_of_metric != 0)
				return set_error(context, ACLB200_ERR_UNSUPPORTED, "calculate_compression_error: the skeleton's object transforms do not fit in shared memory");
		}

		// chunks: runs of jobs of one group whose decoded poses fit the scratch budget (one job at least)
		const uint64_t budget_poses = std::max<uint64_t>(1, context->error_chunk_bytes / std::max<uint64_t>(stride, 1));
		struct Chunk { size_t first_job, num_jobs; uint32_t num_poses; uint32_t rounding; uint32_t metric; };
		std::vector<Chunk> chunks;
		uint64_t max_chunk_poses = 0;
		for (uint32_t pass = 0; pass < 4; ++pass)
		{
			size_t cursor = group_begin[pass];
			while (cursor < group_begin[pass + 1])
			{
				Chunk chunk = { cursor, 0, 0, (pass >> 1) == 0 ? uint32_t(ACLB200_ROUND_NEAREST) : uint32_t(ACLB200_ROUND_NONE), pass & 1u };
				uint64_t poses = 0;
				while (cursor < group_begin[pass + 1] && (chunk.num_jobs == 0 || poses + ordered[cursor].num_samples <= budget_poses))
				{
					ordered[cursor].chunk_first_pose = uint32_t(poses);
					poses += ordered[cursor].num_samples;
					++cursor;
					++chunk.num_jobs;
				}
				if (poses > 0x7FFFFFFFull)
					return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "calculate_compression_error: a single clip has too many samples");
				chunk.num_poses = uint32_t(poses);
				max_chunk_poses = std::max(max_chunk_poses, poses);
				chunks.push_back(chunk);
			}
		}

		// scratch carve-up: jobs | keys | flags | requests | pose jobs | lossy poses
		const size_t jobs_bytes = align_up(sizeof(ErrorJobDev) * ordered.size(), 256);
		const size_t keys_bytes = align_up(sizeof(unsigned long long) * num_jobs, 256);
		const size_t flags_bytes = align_up(sizeof(uint32_t) * num_jobs, 256);
		const size_t requests_bytes = align_up(sizeof(aclb200_request) * size_t(max_chunk_poses), 256);
		const size_t pose_jobs_bytes = align_up(sizeof(uint32_t) * size_t(max_chunk_poses), 256);
		const size_t lossy_bytes = align_up(size_t(max_chunk_poses) * size_t(stride), 256);
		cudaSetDevice(context->device);
		const aclb200_status grown = grow_scratch(context, jobs_bytes + keys_bytes + flags_bytes + requests_bytes + pose_jobs_bytes + lossy_bytes + 256);
		if (grown != ACLB200_OK)
			return grown;
		uint8_t* scratch = static_cast<uint8_t*>(context->d_error_scratch);
		ErrorJobDev* d_jobs = reinterpret_cast<ErrorJobDev*>(scratch);
		unsigned long long* d_keys = reinterpret_cast<unsigned long long*>(scratch + jobs_bytes);
		uint32_t* d_flags = reinterpret_cast<uint32_t*>(scratch + jobs_bytes + keys_bytes);
		aclb200_request* d_requests = reinterpret_cast<aclb200_request*>(scratch + jobs_bytes + keys_bytes + flags_bytes);
		uint32_t* d_pose_jobs = reinterpret_cast<uint32_t*>(scratch + jobs_bytes + keys_bytes + flags_bytes + requests_bytes);
		uint8_t* d_lossy = scratch + jobs_bytes + keys_bytes + flags_bytes + requests_bytes + pose_jobs_bytes;

		cudaStream_t cuda_stream = static_cast<cudaStream_t>(stream);
		const ScratchUse use{ context, cuda_stream };
		cudaError_t error = use.wait();
		// pageable source: the copy has left `ordered` when the call returns
		if (error == cudaSuccess)
			error = cudaMemcpyAsync(d_jobs, ordered.data(), sizeof(ErrorJobDev) * ordered.size(), cudaMemcpyHostToDevice, cuda_stream);
		if (error == cudaSuccess)
			error = cudaMemsetAsync(d_keys, 0, keys_bytes + flags_bytes, cuda_stream);
		if (error != cudaSuccess)
			return check_cuda(context, error, "calculate_compression_error: job upload");

		aclb200_options decode_options = *options;
		decode_options.output_layout = ACLB200_LAYOUT_QVV48;
		decode_options.pose_stride_bytes = stride;
		decode_options.d_request_policies = nullptr;

		for (const Chunk& chunk : chunks)
		{
			if (chunk.num_poses == 0)
				continue;
			ErrorParams p = {};
			p.jobs = d_jobs + chunk.first_job;
			p.num_jobs = uint32_t(chunk.num_jobs);
			p.num_poses = chunk.num_poses;
			p.requests = d_requests;
			p.pose_jobs = d_pose_jobs;
			p.raw_poses = static_cast<const uint8_t*>(d_raw_poses);
			p.lossy_poses = d_lossy;
			p.base_poses = static_cast<const uint8_t*>(d_base_poses);
			p.pose_stride = stride;
			p.parent_indices = d_parent_indices;
			p.shell_distances = d_shell_distances;
			p.output_indices = d_output_indices;
			p.keys = d_keys;
			p.flags = d_flags;
			p.error_matrix = d_out_error_matrix;
			p.error_stride = uint32_t(stride / bone_stride);		// tracks a pose row holds: every job fits (checked above)
			p.plane_stride = plane_stride;
			p.components = components;

			build_error_requests_kernel<<<(chunk.num_poses + 255) / 256, 256, 0, cuda_stream>>>(p);
			error = cudaGetLastError();
			if (error != cudaSuccess)
				return check_cuda(context, error, "calculate_compression_error: request setup");
			context->launch_count++;

			decode_options.rounding_policy = chunk.rounding;
			const aclb200_status decoded = is_transform
				? aclb200_decompress_tracks(context, clipset, d_requests, chunk.num_poses, &decode_options, d_lossy, stream)
				: aclb200_scalar_decompress_tracks(context, clipset, d_requests, chunk.num_poses, &decode_options, d_lossy, stream);
			if (decoded != ACLB200_OK)
				return decoded;

			if (is_transform)
			{
				const uint32_t warps = warps_by_metric[chunk.metric];
				const uint32_t blocks_needed = (chunk.num_poses + warps - 1) / warps;
				const uint32_t blocks = std::min<uint32_t>(blocks_needed, uint32_t(context->num_sms) * 32);
				const size_t smem = size_t(warps) * 2 * (chunk.metric == 1 ? 12u : k_object_components) * plane_stride * sizeof(float);
				if (chunk.metric == 1)
					object_space_kernel<0, 1><<<blocks, warps * 32, smem, cuda_stream>>>(p, ObjectSpaceParams{});
				else
					object_space_kernel<0><<<blocks, warps * 32, smem, cuda_stream>>>(p, ObjectSpaceParams{});
			}
			else
			{
				const uint64_t items = uint64_t(chunk.num_poses) * clipset->info.max_tracks;
				scalar_error_kernel<<<uint32_t((items + 255) / 256), 256, 0, cuda_stream>>>(p, clipset->info.max_tracks);
			}
			error = cudaGetLastError();
			if (error != cudaSuccess)
				return check_cuda(context, error, "calculate_compression_error: error kernel");
			context->launch_count++;
		}

		finalize_error_kernel<<<(num_jobs + 255) / 256, 256, 0, cuda_stream>>>(d_jobs, num_jobs, d_keys, d_flags, d_out_errors);
		error = cudaGetLastError();
		if (error == cudaSuccess)
			context->launch_count++;
		return check_cuda(context, error, "calculate_compression_error");
	}

	// nothing may unwind through the extern "C" boundary: the job tables are host allocations
	aclb200_status aclb200_calculate_compression_error(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_error_job* jobs,
		uint32_t num_jobs, const void* d_raw_poses, const uint32_t* d_parent_indices, const float* d_shell_distances,
		const uint32_t* d_output_indices, const void* d_base_poses, const aclb200_options* options, aclb200_track_error* d_out_errors,
		float* d_out_error_matrix, void* stream)
	{
		if (database_streamed_in(clipset))
			return set_error(context, ACLB200_ERR_UNSUPPORTED, "calculate_compression_error: the clip set's database has chunks streamed in");
		try
		{
			return calculate_compression_error_impl(context, clipset, jobs, num_jobs, d_raw_poses, d_parent_indices, d_shell_distances, d_output_indices,
				d_base_poses, options, d_out_errors, d_out_error_matrix, stream);
		}
		catch (const std::exception&)
		{
			return set_error(context, ACLB200_ERR_OUT_OF_MEMORY, "calculate_compression_error: out of host memory for the job tables");
		}
	}

	static aclb200_status decompress_all_samples_impl(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_error_job* jobs,
		uint32_t num_jobs, const aclb200_options* options, void* d_out, void* stream)
	{
		if (context == nullptr || clipset == nullptr || options == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "null context / clipset / options");
		if (num_jobs == 0)
			return ACLB200_OK;
		if (jobs == nullptr || d_out == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "decompress_all_samples: null jobs / output");
		if (options->d_request_policies != nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "decompress_all_samples builds its own requests: d_request_policies does not apply");

		// the requests of every job, back to back: sample i of a clip at min(i / sample_rate, duration) (convert.impl.h:168)
		std::vector<ErrorJobDev> ordered(num_jobs);
		uint64_t total_poses = 0;
		for (uint32_t index = 0; index < num_jobs; ++index)
		{
			if (jobs[index].clip >= clipset->info.num_clips)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "decompress_all_samples: job names a clip outside the clip set");
			ErrorJobDev dev = {};
			dev.clip = jobs[index].clip;
			dev.num_samples = jobs[index].num_samples;
			dev.sample_rate = jobs[index].sample_rate;
			dev.duration = jobs[index].duration;
			dev.chunk_first_pose = uint32_t(total_poses);
			dev.job_index = index;
			ordered[index] = dev;
			total_poses += jobs[index].num_samples;
		}
		if (total_poses == 0)
			return ACLB200_OK;
		if (total_poses > 0x7FFFFFFFull)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "decompress_all_samples: more than 2^31 poses in one call");

		const size_t jobs_bytes = align_up(sizeof(ErrorJobDev) * ordered.size(), 256);
		const size_t requests_bytes = align_up(sizeof(aclb200_request) * size_t(total_poses), 256);
		const size_t pose_jobs_bytes = align_up(sizeof(uint32_t) * size_t(total_poses), 256);
		cudaSetDevice(context->device);
		const aclb200_status grown = grow_scratch(context, jobs_bytes + requests_bytes + pose_jobs_bytes);
		if (grown != ACLB200_OK)
			return grown;
		uint8_t* scratch = static_cast<uint8_t*>(context->d_error_scratch);
		cudaStream_t cuda_stream = static_cast<cudaStream_t>(stream);
		const ScratchUse use{ context, cuda_stream };
		cudaError_t error = use.wait();
		if (error == cudaSuccess)
			error = cudaMemcpyAsync(scratch, ordered.data(), sizeof(ErrorJobDev) * ordered.size(), cudaMemcpyHostToDevice, cuda_stream);
		if (error != cudaSuccess)
			return check_cuda(context, error, "decompress_all_samples: job upload");

		ErrorParams p = {};
		p.jobs = reinterpret_cast<const ErrorJobDev*>(scratch);
		p.num_jobs = num_jobs;
		p.num_poses = uint32_t(total_poses);
		p.requests = reinterpret_cast<aclb200_request*>(scratch + jobs_bytes);
		p.pose_jobs = reinterpret_cast<uint32_t*>(scratch + jobs_bytes + requests_bytes);
		build_error_requests_kernel<<<(p.num_poses + 255) / 256, 256, 0, cuda_stream>>>(p);
		error = cudaGetLastError();
		if (error != cudaSuccess)
			return check_cuda(context, error, "decompress_all_samples: request setup");
		context->launch_count++;
		return clipset->info.track_type == ACLB200_TRACK_QVVF
			? aclb200_decompress_tracks(context, clipset, p.requests, p.num_poses, options, d_out, stream)
			: aclb200_scalar_decompress_tracks(context, clipset, p.requests, p.num_poses, options, d_out, stream);
	}

	aclb200_status aclb200_decompress_all_samples(aclb200_context* context, const aclb200_clipset* clipset, const aclb200_error_job* jobs,
		uint32_t num_jobs, const aclb200_options* options, void* d_out, void* stream)
	{
		if (database_streamed_in(clipset))
			return set_error(context, ACLB200_ERR_UNSUPPORTED, "decompress_all_samples: the clip set's database has chunks streamed in");
		try
		{
			return decompress_all_samples_impl(context, clipset, jobs, num_jobs, options, d_out, stream);
		}
		catch (const std::exception&)
		{
			return set_error(context, ACLB200_ERR_OUT_OF_MEMORY, "decompress_all_samples: out of host memory for the job table");
		}
	}

	aclb200_status aclb200_set_error_chunk_bytes(aclb200_context* context, uint64_t bytes)
	{
		if (context == nullptr || bytes == 0)
			return ACLB200_ERR_INVALID_ARGUMENT;
		context->error_chunk_bytes = bytes;
		return ACLB200_OK;
	}
}
