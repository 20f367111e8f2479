// acl_b200/csrc/mirror.cu -- left/right mirroring of QVV48 poses already on the device (aclb200_mirror_poses): each row takes its mirror
// row's transform, reflected across the plane normal to the axis and corrected by the row's table entry. One thread per (pose, row); the
// thread of the lower row of each partner pair mirrors both rows, so a pose may be mirrored in place. The row math is obj::mirror_row
// (object_space.cuh), which the mirrored decode (kernels.cu, k_compose_mirror) runs on its staged rows.
#include "object_space.cuh"

namespace aclb200
{
	namespace
	{
		// pose p, row i: mirrored[p] (or 1 without the array) 0 copies the row, 1 mirrors the pair (i, partner(i)) when i is its lower
		// row, any other value writes nothing
		__global__ void __launch_bounds__(256)
		mirror_poses_kernel(const MirrorApply a)
		{
			uint32_t flags = 0;
			const uint64_t num_items = a.num_poses * a.num_rows;
			for (uint64_t item = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; item < num_items; item += uint64_t(gridDim.x) * blockDim.x)
			{
				const uint64_t pose = item / a.num_rows;
				const uint32_t row = uint32_t(item - pose * a.num_rows);
				const uint32_t mirrored = a.mirrored != nullptr ? __ldg(a.mirrored + pose) : 1u;
				const uint8_t* in = a.poses + pose * a.pose_stride;
				uint8_t* out = a.out + pose * a.pose_stride;
				if (mirrored == 0u)
				{
					const float4* src = reinterpret_cast<const float4*>(in + uint64_t(row) * 48);
					const float4 r = src[0], t = src[1], s = src[2];
					float4* dst = reinterpret_cast<float4*>(out + uint64_t(row) * 48);
					dst[0] = r;
					dst[1] = t;
					dst[2] = s;
					continue;
				}
				if (mirrored != 1u)
					continue;
				bool invalid = false;
				const uint32_t partner = obj::mirror_partner(a.table, row, a.num_rows, invalid);
				if (invalid)
					flags |= ACLB200_ERROR_FLAG_INVALID_MIRROR;
				if (partner < row)
					continue;
				obj::mirror_row(out + uint64_t(row) * 48, out + uint64_t(partner) * 48, in + uint64_t(row) * 48, in + uint64_t(partner) * 48,
					a.table + row, a.table + partner, a.axis, false);
			}
			if (flags != 0 && a.flags != nullptr)
				atomicOr(a.flags, flags);
		}
	}

	cudaError_t launch_mirror_poses(const MirrorApply& apply, int num_sms, cudaStream_t stream)
	{
		mirror_poses_kernel<<<pose_operation_blocks(apply.num_poses, apply.num_rows, num_sms), 256, 0, stream>>>(apply);
		return cudaGetLastError();
	}
}
