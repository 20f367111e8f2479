// oracle/ref_object_space.cpp -- TEST INFRASTRUCTURE ONLY: the reference's qvvf_matrix3x4f_transform_error_metric object space on a given
// pose, compiled into _ref/libaclref_object_space.so (oracle/object_space.mk) where the reference tree exists.
#include <acl/compression/transform_error_metrics.h>

#include <cstdint>
#include <vector>

extern "C"
{
	// convert_transforms + local_to_object_space of the unmodified qvvf_matrix3x4f_transform_error_metric (transform_error_metrics.h:397-436)
	// on one pose: local_pose [num_tracks][12] rtm::qvvf rows, parents (0xFFFFFFFF = root, a parent precedes its child), out_object
	// [num_tracks][12] = the xyz lanes of x_axis, y_axis, z_axis, w_axis of each rtm::matrix3x4f. Returns -1 on a parent that does not
	// precede its child, else 0.
	__attribute__((visibility("default"))) int aclref_local_to_object_space_matrix(const float* local_pose, const uint32_t* parents,
		uint32_t num_tracks, float* out_object)
	{
		std::vector<rtm::qvvf> local_qvv(num_tracks);
		std::vector<uint32_t> self(num_tracks);
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
		{
			const float* row = local_pose + size_t(bone) * 12;
			local_qvv[bone] = rtm::qvv_set(rtm::quat_load(row), rtm::vector_load3(row + 4), rtm::vector_load3(row + 8));
			self[bone] = bone;
			if (parents[bone] != acl::k_invalid_track_index && parents[bone] >= bone)
				return -1;
		}
		const acl::qvvf_matrix3x4f_transform_error_metric error_metric;
		std::vector<rtm::matrix3x4f> local(num_tracks), object(num_tracks);
		acl::itransform_error_metric::convert_transforms_args convert_args;
		convert_args.dirty_transform_indices = self.data();
		convert_args.num_dirty_transforms = num_tracks;
		convert_args.transforms = local_qvv.data();
		convert_args.num_transforms = num_tracks;
		convert_args.sample_index = 0;
		convert_args.is_additive_base = false;
		convert_args.is_lossy = false;
		error_metric.convert_transforms(convert_args, local.data());
		acl::itransform_error_metric::local_to_object_space_args object_args;
		object_args.dirty_transform_indices = self.data();
		object_args.num_dirty_transforms = num_tracks;
		object_args.parent_transform_indices = parents;
		object_args.local_transforms = local.data();
		object_args.num_transforms = num_tracks;
		error_metric.local_to_object_space(object_args, object.data());
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
		{
			float* row = out_object + size_t(bone) * 12;
			rtm::vector_store3(object[bone].x_axis, row + 0);
			rtm::vector_store3(object[bone].y_axis, row + 3);
			rtm::vector_store3(object[bone].z_axis, row + 6);
			rtm::vector_store3(object[bone].w_axis, row + 9);
		}
		return 0;
	}
}
