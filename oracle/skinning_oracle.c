/* oracle/skinning_oracle.c -- TEST INFRASTRUCTURE ONLY: the port's skinning matrices as entry points of their own, built into
 * liboracle_skinning.so by oracle/skinning.mk. The restatements it needs (rtm_matrix_mul and the matrix walk of
 * qvvf_matrix3x4f_transform_error_metric) are file-local to acl_oracle.c, so that file is compiled in here unchanged. */
#include "acl_oracle.c"

/* skin = rtm::matrix_mul(inverse_bind, object) (matrix3x4f.h:298-321) on every bone: object and inverse_bind [num_tracks][4][3] (x_axis,
 * y_axis, z_axis, w_axis, xyz each), out [num_tracks][3][4] as the library stores it: row c = (x_axis[c], y_axis[c], z_axis[c], w_axis[c]) */
void aclo_skin_object_matrices(const float* object_pose, const float* inverse_bind, uint32_t num_tracks, float* out_rows)
{
	for (uint32_t bone = 0; bone < num_tracks; ++bone)
	{
		float inverse[4][3], object[4][3], skin[4][3];
		memcpy(inverse, inverse_bind + (size_t)bone * 12, sizeof(inverse));
		memcpy(object, object_pose + (size_t)bone * 12, sizeof(object));
		rtm_matrix_mul(inverse, object, skin);
		float* rows = out_rows + (size_t)bone * 12;
		for (int c = 0; c < 3; ++c)
			for (int axis = 0; axis < 4; ++axis)
				rows[c * 4 + axis] = skin[axis][c];
	}
}

/* convert_transforms + local_to_object_space of qvvf_matrix3x4f_transform_error_metric (transform_error_metrics.h:397-436), then the
 * skinning step above: rtm::qvvf rows of 12 floats in, skinning rows out. Returns -1 when a parent does not precede its child, else 0. */
int aclo_local_to_skinning(const float* local_pose, const uint32_t* parent_indices, const float* inverse_bind, uint32_t num_tracks, float* out_rows)
{
	float* object = (float*)malloc((size_t)num_tracks * 12 * sizeof(float) + 1);
	const int result = matrix_local_to_object_space(local_pose, parent_indices, num_tracks, object);
	if (result == 0)
		aclo_skin_object_matrices(object, inverse_bind, num_tracks, out_rows);
	free(object);
	return result;
}
