/* oracle/root_motion_oracle.c -- TEST INFRASTRUCTURE ONLY: the port's root motion (aclb200_extract_root_motion) given the root rows, built
 * into liboracle_root_motion.so by oracle/root_motion.mk. The restatements it needs (qvv_mul_plain with its negative scale branch,
 * rtm_quat_mul_vector3) are file-local to acl_oracle.c, so that file is compiled in here unchanged. Rows are rtm::qvvf rows of 12 floats
 * (rotation xyzw, translation xyz + w, scale xyz + w); the rows written carry 0 in both w lanes. */
#include "acl_oracle.c"

/* rtm::qvv_inverse(input), qvvf.h:389-395, the one argument form: quat_conjugate (sign bits of x, y, z xor-ed, quatf.h:482-491),
 * vector_reciprocal = 1 / scale (_mm_div_ps, vector4f.h:1310), translation = -quat_mul_vector3(translation * inv_scale, inv_rotation)
 * (vector_neg xors the sign bits, vector4f.h:1261-1271) */
static void qvv_inverse(const float in[12], float out[12])
{
	float result[12];
	for (int i = 0; i < 3; ++i)
		result[i] = u32_as_f32(f32_as_u32(in[i]) ^ 0x80000000u);
	result[3] = in[3];
	for (int i = 0; i < 3; ++i)
		result[8 + i] = 1.0f / in[8 + i];
	const float scaled[3] = { in[4] * result[8], in[5] * result[9], in[6] * result[10] };
	float rotated[3];
	rtm_quat_mul_vector3(scaled, result, rotated);
	for (int i = 0; i < 3; ++i)
		result[4 + i] = u32_as_f32(f32_as_u32(rotated[i]) ^ 0x80000000u);
	result[7] = 0.0f;
	result[11] = 0.0f;
	memcpy(out, result, sizeof(result));
}

void aclo_qvv_inverse(const float* in, float* out)
{
	qvv_inverse(in, out);
}

void aclo_qvv_mul(const float* lhs, const float* rhs, int normalize_mode, float* out)
{
	qvv_mul_plain(lhs, rhs, normalize_mode, out);
}

/* rel(a, b) = qvv_mul(T(b), qvv_inverse(T(a))): the delta with T(b) = qvv_mul(delta, T(a)) */
static int relative(const float a[12], const float b[12], int normalize_mode, float out[12])
{
	float inverse[12];
	qvv_inverse(a, inverse);
	return qvv_mul_plain(b, inverse, normalize_mode, out);
}

/* M of one request from its four root samples T(from), T(to), T(D) (`end`), T(0) (`start`):
 *   cycles == 0: rel(from, to);
 *   k > 0: rel(from, D), then k - 1 times M = qvv_mul(rel(0, D), M), then M = qvv_mul(rel(0, to), M);
 *   k < 0: rel(from, 0), then -k - 1 times M = qvv_mul(rel(D, 0), M), then M = qvv_mul(rel(D, to), M).
 * normalize_mode: the flavour of quat_from_matrix's closing normalisation on qvv_mul's negative scale branch (0: the reference's rsqrtss +
 * 2 Newton-Raphson steps, 1: IEEE 1 / sqrt as the CUDA path). Returns 1 when a qvv_mul took the negative scale branch. */
int aclo_root_motion(const float* from, const float* to, const float* end, const float* start, int32_t cycles, int normalize_mode, float* out)
{
	float motion[12];
	int negative = 0;
	if (cycles == 0)
		negative |= relative(from, to, normalize_mode, motion);
	else
	{
		const float* reached = cycles > 0 ? end : start;
		const float* resumed = cycles > 0 ? start : end;
		float cycle[12], last[12];
		negative |= relative(from, reached, normalize_mode, motion);
		negative |= relative(resumed, reached, normalize_mode, cycle);
		const int32_t full_cycles = (cycles > 0 ? cycles : -cycles) - 1;
		for (int32_t i = 0; i < full_cycles; ++i)
			negative |= qvv_mul_plain(cycle, motion, normalize_mode, motion);
		negative |= relative(resumed, to, normalize_mode, last);
		negative |= qvv_mul_plain(last, motion, normalize_mode, motion);
	}
	memcpy(out, motion, sizeof(motion));
	return negative;
}
