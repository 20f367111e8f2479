// oracle/ref_skinning.cpp -- TEST INFRASTRUCTURE ONLY: skinning matrices from the unmodified reference, compiled into
// _ref/libaclref_skinning.so (oracle/skinning.mk) where the reference tree exists. The object space is ref_object_space.cpp's (the metric's
// own convert_transforms + local_to_object_space), compiled in here unchanged; the skinning step is rtm::matrix_mul(inverse_bind, object).
#include "ref_object_space.cpp"

#include <rtm/matrix3x4f.h>

namespace
{
	rtm::matrix3x4f load_matrix(const float* axes)
	{
		return rtm::matrix_set(rtm::vector_load3(axes + 0), rtm::vector_load3(axes + 3), rtm::vector_load3(axes + 6), rtm::vector_load3(axes + 9));
	}

	// skin[b] = rtm::matrix_mul(inverse_bind[b], object[b]) of every bone, or an empty vector when a parent does not precede its child
	std::vector<rtm::matrix3x4f> skinning_matrices(const float* local_pose, const uint32_t* parents, const float* inverse_bind, uint32_t num_tracks)
	{
		std::vector<float> object(size_t(num_tracks) * 12);
		if (aclref_local_to_object_space_matrix(local_pose, parents, num_tracks, object.data()) != 0)
			return {};
		std::vector<rtm::matrix3x4f> skin;
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
			skin.push_back(rtm::matrix_mul(load_matrix(inverse_bind + size_t(bone) * 12), load_matrix(object.data() + size_t(bone) * 12)));
		return skin;
	}
}

extern "C"
{
	// local_pose [num_tracks][12] rtm::qvvf rows, inverse_bind [num_tracks][4][3] (x_axis, y_axis, z_axis, w_axis, xyz each), out_rows
	// [num_tracks][3][4]: row c = (x_axis[c], y_axis[c], z_axis[c], w_axis[c]) of skin. Returns -1 on a parent that does not precede its
	// child, else 0.
	__attribute__((visibility("default"))) int aclref_local_to_skinning(const float* local_pose, const uint32_t* parents, const float* inverse_bind,
		uint32_t num_tracks, float* out_rows)
	{
		const std::vector<rtm::matrix3x4f> skin = skinning_matrices(local_pose, parents, inverse_bind, num_tracks);
		if (skin.size() != num_tracks)
			return -1;
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
		{
			float axes[4][3];
			rtm::vector_store3(skin[bone].x_axis, axes[0]);
			rtm::vector_store3(skin[bone].y_axis, axes[1]);
			rtm::vector_store3(skin[bone].z_axis, axes[2]);
			rtm::vector_store3(skin[bone].w_axis, axes[3]);
			for (int c = 0; c < 3; ++c)
				for (int axis = 0; axis < 4; ++axis)
					out_rows[size_t(bone) * 12 + c * 4 + axis] = axes[axis][c];
		}
		return 0;
	}

	// rtm::matrix_mul_point3(points[b], skin[b]) (matrix3x4f.h:326-336) of every bone into out_points [num_tracks][3]
	__attribute__((visibility("default"))) int aclref_skinned_points(const float* local_pose, const uint32_t* parents, const float* inverse_bind,
		uint32_t num_tracks, const float* points, float* out_points)
	{
		const std::vector<rtm::matrix3x4f> skin = skinning_matrices(local_pose, parents, inverse_bind, num_tracks);
		if (skin.size() != num_tracks)
			return -1;
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
			rtm::vector_store3(rtm::matrix_mul_point3(rtm::vector_load3(points + size_t(bone) * 3), skin[bone]), out_points + size_t(bone) * 3);
		return 0;
	}
}
