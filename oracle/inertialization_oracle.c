/* oracle/inertialization_oracle.c -- TEST INFRASTRUCTURE ONLY: the inertialization capture and apply (aclb200_begin_inertialization,
 * aclb200_inertialize_poses) restated on the CPU, built into liboracle_inertialization.so by oracle/inertialization.mk. rtm's
 * quat_rotation_log and quat_rotation_exp (quatf.h:1306-1375) are restated from their SSE2 paths, with the scalar_acos, scalar_sin and
 * scalar_cos polynomials they call (scalarf.h:855-967, 1142-1174) written in plain float arithmetic (the build passes -ffp-contract=off).
 * rtm_quat_mul is file-local to acl_oracle.c, so that file is compiled in here unchanged. */
#include "acl_oracle.c"

#include <math.h>

/* rtm's constants are static_cast<float> of double literals (constants.h:35-47) */
static const float k_pi = (float)3.141592653589793238462643383279502884;
static const float k_half_pi = (float)1.570796326794896619231321691639751442;
static const float k_two_pi = (float)6.283185307179586476925286766559005768;
static const float k_one_div_two_pi = (float)1.591549430918953357688837633725143620e-01;

static float or_sign(float v, uint32_t sign) { return u32_as_f32(f32_as_u32(v) | sign); }

/* rtm::scalar_acos (SSE2 path) */
static float rtm_acos(float v)
{
	const float x = fabsf(v);
	float r = (x * -1.2690614339589956e-3F) + 6.7072304676685235e-3F;
	r = (r * x) - 1.7162031184398074e-2F;
	r = (r * x) + 3.0961594977611639e-2F;
	r = (r * x) - 5.0207843052845647e-2F;
	r = (r * x) + 8.8986946573346160e-2F;
	r = (r * x) - 2.1459960076929829e-1F;
	r = (r * x) + 1.5707963267948966F;
	r = r * sqrtf(1.0f - x);
	if (v < 0.0f)
		r = k_pi - r;
	return r;
}

/* the range reduction of scalar_sin / scalar_cos: banker's rounding (roundss, nearbyintf in the default rounding mode), then the
 * reflection about copysign(pi, x) when |x| <= pi / 2 is false */
static float reduce_angle(float angle, int* within_half_pi)
{
	float x = angle - nearbyintf(angle * k_one_div_two_pi) * k_two_pi;
	const float reference = or_sign(k_pi, f32_as_u32(x) & 0x80000000u);
	*within_half_pi = fabsf(x) <= k_half_pi;
	return *within_half_pi ? x : reference - x;
}

static float rtm_sin(float angle)
{
	int within;
	const float x = reduce_angle(angle, &within);
	const float x2 = x * x;
	float r = (x2 * -2.3828544692960918e-8F) + 2.7521557770526783e-6F;
	r = (r * x2) - 1.9840782426250314e-4F;
	r = (r * x2) + 8.3333303183525942e-3F;
	r = (r * x2) - 1.6666666601721269e-1F;
	r = (r * x2) + 1.0F;
	return r * x;
}

static float rtm_cos(float angle)
{
	int within;
	const float x = reduce_angle(angle, &within);
	const float x2 = x * x;
	float r = (x2 * -2.6051615464872668e-7F) + 2.4760495088926859e-5F;
	r = (r * x2) - 1.3888377661039897e-3F;
	r = (r * x2) + 4.1666638865338612e-2F;
	r = (r * x2) - 4.9999999508695869e-1F;
	r = (r * x2) + 1.0F;
	return within ? r : or_sign(r, 0x80000000u);
}

/* rtm::quat_rotation_log(q), w written as 0 */
void aclo_quat_rotation_log(const float q[4], float out[4])
{
	const float lower = q[3] > -1.0f ? q[3] : -1.0f;		/* _mm_max_ss(w, -1): NaN gives -1 */
	const float w = lower < 1.0f ? lower : 1.0f;			/* _mm_min_ss(., 1) */
	const float half_angle = rtm_acos(w);
	const float inv_len = 1.0f / sqrtf((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]);
	const float s = inv_len * half_angle;
	const int near_identity = w > 1.0f - 1.0e-6f;
	for (int i = 0; i < 3; ++i)
		out[i] = near_identity ? q[i] : q[i] * s;
	out[3] = 0.0f;
}

/* rtm::quat_rotation_exp(v) of v's xyz (its w is not read) */
void aclo_quat_rotation_exp(const float v[4], float out[4])
{
	const float len = sqrtf((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
	const float sine = rtm_sin(len);
	const int near_zero = len < 1.0e-6f;
	for (int i = 0; i < 3; ++i)
		out[i] = near_zero ? v[i] : (v[i] / len) * sine;
	out[3] = rtm_cos(len);
}

/* 2 log(abs(quat_mul(conj(from), to))).xyz */
static void scaled_angle_axis_between(const float from[4], const float to[4], float out[3])
{
	const float conj[4] = { -from[0], -from[1], -from[2], from[3] };
	float q[4], l[4];
	rtm_quat_mul(conj, to, q);
	if (q[3] < 0.0f)
		for (int i = 0; i < 4; ++i)
			q[i] = -q[i];
	aclo_quat_rotation_log(q, l);
	for (int i = 0; i < 3; ++i)
		out[i] = 2.0f * l[i];
}

/* aclb200_begin_inertialization on one transition: [num_tracks][12] QVV48 rows in, [num_tracks][16] record entries out (rot_x, rot_v,
 * pos_x, pos_v, each xyz + 0) */
void aclo_begin_inertialization(const float* src, const float* src_prev, const float* dst, const float* dst_prev, uint32_t num_tracks,
	float inv_dt, float* record)
{
	for (uint32_t bone = 0; bone < num_tracks; ++bone)
	{
		const float* s = src + (size_t)bone * 12;
		const float* sp = src_prev + (size_t)bone * 12;
		const float* d = dst + (size_t)bone * 12;
		const float* dp = dst_prev + (size_t)bone * 12;
		float* e = record + (size_t)bone * 16;
		float rot_x[3], src_w[3], dst_w[3];
		scaled_angle_axis_between(d, s, rot_x);
		scaled_angle_axis_between(sp, s, src_w);
		scaled_angle_axis_between(dp, d, dst_w);
		for (int i = 0; i < 3; ++i)
		{
			e[i] = rot_x[i];
			e[4 + i] = src_w[i] * inv_dt - dst_w[i] * inv_dt;
			e[8 + i] = s[4 + i] - d[4 + i];
			e[12 + i] = (s[4 + i] - sp[4 + i]) * inv_dt - (d[4 + i] - dp[4 + i]) * inv_dt;
		}
		e[3] = e[7] = e[11] = e[15] = 0.0f;
	}
}

/* the spring of one pose: y, e */
void aclo_inertialization_decay(float elapsed, float halflife, float out[2])
{
	const float y = (2.7725887f / (halflife + 1e-5f)) * 0.5f;
	const float u = y * elapsed;
	out[0] = y;
	out[1] = 1.0f / (((1.0f + u) + (0.48f * u) * u) + ((0.235f * u) * u) * u);
}

/* aclb200_inertialize_poses on one pose with one record: [num_tracks][12] rows in and out (out may be pose) */
void aclo_inertialize_pose(const float* pose, const float* record, uint32_t num_tracks, float elapsed, float halflife, float* out)
{
	float decay[2];
	aclo_inertialization_decay(elapsed, halflife, decay);
	const float y = decay[0], e = decay[1];
	for (uint32_t bone = 0; bone < num_tracks; ++bone)
	{
		const float* d = pose + (size_t)bone * 12;
		const float* r = record + (size_t)bone * 16;
		float half_offset[4] = { 0.0f, 0.0f, 0.0f, 0.0f }, offset_q[4], row[12];
		for (int i = 0; i < 3; ++i)
		{
			half_offset[i] = (e * (r[i] + (r[4 + i] + r[i] * y) * elapsed)) * 0.5f;
			row[4 + i] = d[4 + i] + e * (r[8 + i] + (r[12 + i] + r[8 + i] * y) * elapsed);
			row[8 + i] = d[8 + i];
		}
		aclo_quat_rotation_exp(half_offset, offset_q);
		rtm_quat_mul(d, offset_q, row);
		row[7] = 0.0f;
		row[11] = 0.0f;
		memcpy(out + (size_t)bone * 12, row, sizeof(row));
	}
}
