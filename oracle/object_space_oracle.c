/* oracle/object_space_oracle.c -- TEST INFRASTRUCTURE ONLY: the port's matrix object space as an entry point of its own, built into
 * liboracle_object_space.so by oracle/object_space.mk. The restatements it needs (rtm_matrix_from_qvv, rtm_matrix_mul and the walk of
 * qvvf_matrix3x4f_transform_error_metric) are file-local to acl_oracle.c, so that file is compiled in here unchanged. */
#include "acl_oracle.c"

/* convert_transforms + local_to_object_space of qvvf_matrix3x4f_transform_error_metric (transform_error_metrics.h:397-436): rtm::qvvf rows
 * of 12 floats in, [num_tracks][4][3] out (x_axis, y_axis, z_axis, w_axis, xyz each). Returns -1 when a parent does not precede its child,
 * else 0. */
int aclo_local_to_object_space_matrix(const float* local_pose, const uint32_t* parent_indices, uint32_t num_tracks, float* out_object_pose)
{
	return matrix_local_to_object_space(local_pose, parent_indices, num_tracks, out_object_pose);
}
