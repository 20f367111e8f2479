// acl_b200/csrc/inertialization.cu -- inertialized transitions between clips: the capture (aclb200_begin_inertialization) records each
// bone's offset from the displayed pose to the destination pose, with the offset's velocity; the apply (aclb200_inertialize_poses) decays
// that offset onto poses already on the device. Both run one thread per (pose, bone) on QVV48 rows, with the device functions of
// object_space.cuh (capture_inertialization_row, inertialize_row): rtm's quat_rotation_log / quat_rotation_exp and quat_mul in unfused
// IEEE operations.
#include "object_space.cuh"

namespace aclb200
{
	namespace
	{
		// transition j, bone b: the record entry at records + slot(j) * record_stride + b * 64, slot(j) = record_slots[j] or j
		__global__ void __launch_bounds__(256)
		begin_inertialization_kernel(const InertializationCapture c)
		{
			const uint64_t num_items = c.num_transitions * c.num_tracks;
			for (uint64_t item = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; item < num_items; item += uint64_t(gridDim.x) * blockDim.x)
			{
				const uint64_t transition = item / c.num_tracks;
				const uint32_t bone = uint32_t(item - transition * c.num_tracks);
				const uint64_t row = transition * c.pose_stride + uint64_t(bone) * 48;
				const uint64_t slot = c.record_slots != nullptr ? __ldg(c.record_slots + transition) : transition;
				float4* entry = reinterpret_cast<float4*>(c.records + slot * c.record_stride + uint64_t(bone) * 64);
				obj::capture_inertialization_row(entry, reinterpret_cast<const float4*>(c.src + row), reinterpret_cast<const float4*>(c.src_prev + row),
					reinterpret_cast<const float4*>(c.dst + row), reinterpret_cast<const float4*>(c.dst_prev + row), c.inv_dt);
			}
		}

		// pose p, bone b: inertializations[p] names the record; ACLB200_NO_INERTIALIZATION copies the row unchanged, a record at or above
		// num_records writes nothing. out may be poses: a thread reads its row before it writes it.
		__global__ void __launch_bounds__(256)
		inertialize_poses_kernel(const InertializationApply a)
		{
			const uint64_t num_items = a.num_poses * a.num_tracks;
			for (uint64_t item = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; item < num_items; item += uint64_t(gridDim.x) * blockDim.x)
			{
				const uint64_t pose = item / a.num_tracks;
				const uint32_t bone = uint32_t(item - pose * a.num_tracks);
				const uint64_t offset = pose * a.pose_stride + uint64_t(bone) * 48;
				const float4* row = reinterpret_cast<const float4*>(a.poses + offset);
				float4* out_row = reinterpret_cast<float4*>(a.out + offset);
				const aclb200_inertialization inertialization = a.inertializations[pose];
				if (inertialization.record == ACLB200_NO_INERTIALIZATION)
				{
					const float4 r = row[0], t = row[1], s = row[2];
					out_row[0] = r;
					out_row[1] = t;
					out_row[2] = s;
					continue;
				}
				if (inertialization.record >= a.num_records)
					continue;
				const float4* entry = reinterpret_cast<const float4*>(a.records + uint64_t(inertialization.record) * a.record_stride + uint64_t(bone) * 64);
				obj::inertialize_row(a.out + offset, a.poses + offset, entry, obj::inertialization_decay(inertialization.elapsed,
					inertialization.halflife), false);
			}
		}
	}

	cudaError_t launch_begin_inertialization(const InertializationCapture& capture, int num_sms, cudaStream_t stream)
	{
		begin_inertialization_kernel<<<pose_operation_blocks(capture.num_transitions, capture.num_tracks, num_sms), 256, 0, stream>>>(capture);
		return cudaGetLastError();
	}

	cudaError_t launch_inertialize_poses(const InertializationApply& apply, int num_sms, cudaStream_t stream)
	{
		inertialize_poses_kernel<<<pose_operation_blocks(apply.num_poses, apply.num_tracks, num_sms), 256, 0, stream>>>(apply);
		return cudaGetLastError();
	}
}
