// acl_b200/csrc/object_space.cuh -- the hierarchy walk shared by the error measurement (error_metric.cu: object_space_kernel), the object
// space decode (kernels.cu: transform_decompress_tracks_kernel<..., COMPOSE = k_compose_object>) and the bone query (bones.cu, the walk
// restricted to the ancestor closure of the listed bones): the reference's
// qvv and 3x4 matrix operations in unfused IEEE operations, and the wavefront loop one warp runs over a pose. Also acl::apply_additive_to_base, which
// the error measurement, the additive decode (COMPOSE = k_compose_additive) and aclb200_apply_additive_to_base share, and rtm::qvv_lerp, which
// the blend decode (COMPOSE = k_compose_blend) and aclb200_blend_poses share. And the skinning step, which the three composed decodes (with
// the internal object kind k_object_skinning) and aclb200_local_to_skinning run after the matrix walk. And rtm::qvv_inverse, which root motion
// (root_motion.cu) composes with qvv_mul, and root motion's composition for the pose features (features.cu).
//
// The wavefront loop: a warp takes 32 consecutive bones at a time; a lane whose parent lies in an earlier chunk -- or was finished by an
// earlier wavefront of this chunk -- computes, the others wait for the next wavefront (skeletons are shallow and bushy: a handful of
// wavefronts per chunk). A bone's local transform sits in the slot its object transform will take.
#pragma once

#include "context.h"

#include <type_traits>

namespace aclb200
{
	namespace obj
	{
		namespace
		{
			constexpr uint32_t k_invalid_track = 0xFFFFFFFFu;			// acl::k_invalid_track_index, core/track_types.h
			constexpr uint32_t k_object_components = 10;				// rotation xyzw, translation xyz, scale xyz

			// ---- the reference's float operations, spelled out so nothing can be contracted -------------------------------------------
			// The measurement runs the SAME operation sequence on the raw and on the lossy pose: the two travel as one f32x2 pair
			// (x = raw, y = lossy). Each operation is one scalar __fmul_rn / __fadd_rn / __fsub_rn per lane, intrinsics that are never
			// contracted into an FMA. Signs: the reference xors sign masks into products and adds them; -(p) + q == q - p, p + -(q) == p - q
			// and -(p) + -(q) == -(p + q) hold exactly in IEEE arithmetic, so the sums below are written with subtractions and no negation.
			template<class V> struct Fp;

			template<> struct Fp<float>
			{
				__device__ __forceinline__ float mul(float a, float b) const { return __fmul_rn(a, b); }
				__device__ __forceinline__ float add(float a, float b) const { return __fadd_rn(a, b); }
				__device__ __forceinline__ float sub(float a, float b) const { return __fsub_rn(a, b); }
				__device__ __forceinline__ float splat(float a) const { return a; }
				__device__ __forceinline__ float inv_sqrt(float a) const { return __fdiv_rn(1.0f, __fsqrt_rn(a)); }
				__device__ __forceinline__ bool any_negative(float a, float b) const { return fminf(a, b) < 0.0f; }
			};

			template<> struct Fp<float2>
			{
				__device__ __forceinline__ float2 mul(float2 a, float2 b) const { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
				__device__ __forceinline__ float2 add(float2 a, float2 b) const { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
				__device__ __forceinline__ float2 sub(float2 a, float2 b) const { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
				__device__ __forceinline__ float2 splat(float a) const { return make_float2(a, a); }
				__device__ __forceinline__ float2 inv_sqrt(float2 a) const { return make_float2(__fdiv_rn(1.0f, __fsqrt_rn(a.x)), __fdiv_rn(1.0f, __fsqrt_rn(a.y))); }
				__device__ __forceinline__ bool any_negative(float2 a, float2 b) const { return fminf(a.x, b.x) < 0.0f || fminf(a.y, b.y) < 0.0f; }
			};

			template<class V> struct Quat { V x, y, z, w; };
			template<class V> struct Vec3 { V x, y, z; };
			template<class V> struct Qvv { Quat<V> rotation; Vec3<V> translation; Vec3<V> scale; };

			// rtm::quat_mul, external/rtm/includes/rtm/quatf.h:498-545 (SSE2 path): (rw*l + s0*(rx*l_wzyx)) + (s1*(ry*l_zwxy) + s2*(rz*l_yxwz))
			template<class V>
			__device__ __forceinline__ Quat<V> quat_mul(const Fp<V>& fp, const Quat<V>& l, const Quat<V>& r)
			{
				Quat<V> out;
				out.x = fp.add(fp.add(fp.mul(r.w, l.x), fp.mul(r.x, l.w)), fp.sub(fp.mul(r.y, l.z), fp.mul(r.z, l.y)));
				out.y = fp.add(fp.sub(fp.mul(r.w, l.y), fp.mul(r.x, l.z)), fp.add(fp.mul(r.y, l.w), fp.mul(r.z, l.x)));
				out.z = fp.add(fp.add(fp.mul(r.w, l.z), fp.mul(r.x, l.y)), fp.sub(fp.mul(r.z, l.w), fp.mul(r.y, l.x)));
				out.w = fp.sub(fp.sub(fp.mul(r.w, l.w), fp.mul(r.x, l.x)), fp.add(fp.mul(r.y, l.y), fp.mul(r.z, l.z)));
				return out;
			}

			// rtm::quat_mul_vector3, quatf.h:616-668 (SSE2 path): temp = conjugate(r) * (v, 0) without its W terms, result = temp * r
			template<class V>
			__device__ __forceinline__ Vec3<V> quat_mul_vector3(const Fp<V>& fp, const Vec3<V>& v, const Quat<V>& r)
			{
				const V t0 = fp.add(fp.sub(fp.mul(v.x, r.w), fp.mul(v.y, r.z)), fp.mul(v.z, r.y));
				const V t1 = fp.sub(fp.add(fp.mul(v.x, r.z), fp.mul(v.y, r.w)), fp.mul(v.z, r.x));
				const V t2 = fp.add(fp.sub(fp.mul(v.y, r.x), fp.mul(v.x, r.y)), fp.mul(v.z, r.w));
				const V t3 = fp.add(fp.add(fp.mul(v.x, r.x), fp.mul(v.y, r.y)), fp.mul(v.z, r.z));
				Vec3<V> out;
				out.x = fp.add(fp.add(fp.mul(r.w, t0), fp.mul(r.x, t3)), fp.sub(fp.mul(r.y, t2), fp.mul(r.z, t1)));
				out.y = fp.add(fp.sub(fp.mul(r.w, t1), fp.mul(r.x, t2)), fp.add(fp.mul(r.y, t3), fp.mul(r.z, t0)));
				out.z = fp.add(fp.add(fp.mul(r.w, t2), fp.mul(r.x, t1)), fp.sub(fp.mul(r.z, t3), fp.mul(r.y, t0)));
				return out;
			}

			// rtm::quat_normalize, quatf.h:917-953: dot = (x2 + z2) + (y2 + w2); IEEE 1 / sqrt in place of the rsqrtss + 2 Newton-Raphson steps
			template<class V>
			__device__ __forceinline__ Quat<V> quat_normalize(const Fp<V>& fp, const Quat<V>& q)
			{
				const V dot = fp.add(fp.add(fp.mul(q.x, q.x), fp.mul(q.z, q.z)), fp.add(fp.mul(q.y, q.y), fp.mul(q.w, q.w)));
				const V inv_len = fp.inv_sqrt(dot);
				Quat<V> out;
				out.x = fp.mul(q.x, inv_len);
				out.y = fp.mul(q.y, inv_len);
				out.z = fp.mul(q.z, inv_len);
				out.w = fp.mul(q.w, inv_len);
				return out;
			}

			// ---- the negative scale branch of rtm::qvv_mul (qvvf.h:320-345): through matrices. Rare (mirrored bones), data dependent branches
			// (quat_from_matrix), so it runs per stream on plain floats, out of line: matrix_from_qvv (matrix3x4f.h:134-159), matrix_mul (:298-321,
			// vector_mul_add = (v0 * v1) + v2 on SSE2), matrix_remove_scale (:636-644 = vector_normalize3(axis, axis, 1e-8), vector4f.h:2310-2318),
			// the result scale's sign bits xor-ed onto the axes, quat_from_matrix (impl/matrix_affine_common.h:153-227, its closing
			// quat_normalize with the IEEE 1 / sqrt like every normalisation here) ----
			struct Matrix3x4 { float m[4][3]; };

			__device__ __forceinline__ Matrix3x4 matrix_from_qvv(const Qvv<float>& q)
			{
				const Fp<float> fp{};
				const float x2 = fp.add(q.rotation.x, q.rotation.x), y2 = fp.add(q.rotation.y, q.rotation.y), z2 = fp.add(q.rotation.z, q.rotation.z);
				const float xx = fp.mul(q.rotation.x, x2), xy = fp.mul(q.rotation.x, y2), xz = fp.mul(q.rotation.x, z2);
				const float yy = fp.mul(q.rotation.y, y2), yz = fp.mul(q.rotation.y, z2), zz = fp.mul(q.rotation.z, z2);
				const float wx = fp.mul(q.rotation.w, x2), wy = fp.mul(q.rotation.w, y2), wz = fp.mul(q.rotation.w, z2);
				Matrix3x4 out;
				out.m[0][0] = fp.mul(fp.sub(1.0f, fp.add(yy, zz)), q.scale.x);	out.m[0][1] = fp.mul(fp.add(xy, wz), q.scale.x);				out.m[0][2] = fp.mul(fp.sub(xz, wy), q.scale.x);
				out.m[1][0] = fp.mul(fp.sub(xy, wz), q.scale.y);				out.m[1][1] = fp.mul(fp.sub(1.0f, fp.add(xx, zz)), q.scale.y);	out.m[1][2] = fp.mul(fp.add(yz, wx), q.scale.y);
				out.m[2][0] = fp.mul(fp.add(xz, wy), q.scale.z);				out.m[2][1] = fp.mul(fp.sub(yz, wx), q.scale.z);				out.m[2][2] = fp.mul(fp.sub(1.0f, fp.add(xx, yy)), q.scale.z);
				out.m[3][0] = q.translation.x;									out.m[3][1] = q.translation.y;									out.m[3][2] = q.translation.z;
				return out;
			}

			__device__ __noinline__ void qvv_mul_negative_scale(const Qvv<float>* lhs_in, const Qvv<float>* rhs_in, Qvv<float>* out)
			{
				const Fp<float> fp{};
				const Qvv<float> lhs = *lhs_in, rhs = *rhs_in;
				const Matrix3x4 l = matrix_from_qvv(lhs), r = matrix_from_qvv(rhs);
				float m[4][3];
				#pragma unroll
				for (int row = 0; row < 4; ++row)
					#pragma unroll
					for (int c = 0; c < 3; ++c)
					{
						float tmp = fp.mul(l.m[row][0], r.m[0][c]);
						tmp = fp.add(fp.mul(l.m[row][1], r.m[1][c]), tmp);
						tmp = fp.add(fp.mul(l.m[row][2], r.m[2][c]), tmp);
						m[row][c] = row == 3 ? fp.add(r.m[3][c], tmp) : tmp;
					}
				const float scale[3] = { fp.mul(lhs.scale.x, rhs.scale.x), fp.mul(lhs.scale.y, rhs.scale.y), fp.mul(lhs.scale.z, rhs.scale.z) };
				#pragma unroll
				for (int axis = 0; axis < 3; ++axis)
				{
					const float len_sq = fp.add(fp.add(fp.mul(m[axis][0], m[axis][0]), fp.mul(m[axis][1], m[axis][1])), fp.mul(m[axis][2], m[axis][2]));
					const float inv_len = len_sq >= 1.0e-8f ? fp.inv_sqrt(len_sq) : 1.0f;
					const uint32_t sign = __float_as_uint(scale[axis]) & 0x80000000u;
					#pragma unroll
					for (int c = 0; c < 3; ++c)
					{
						const float normalized = len_sq >= 1.0e-8f ? fp.mul(m[axis][c], inv_len) : m[axis][c];
						m[axis][c] = __uint_as_float(__float_as_uint(normalized) ^ sign);
					}
				}

				Quat<float> q;
				bool zero_axis = false;
				#pragma unroll
				for (int axis = 0; axis < 3; ++axis)
					zero_axis = zero_axis || (fabsf(m[axis][0]) <= 0.00001f && fabsf(m[axis][1]) <= 0.00001f && fabsf(m[axis][2]) <= 0.00001f);
				const float trace = fp.add(fp.add(m[0][0], m[1][1]), m[2][2]);
				if (zero_axis)
					q = Quat<float>{ 0.0f, 0.0f, 0.0f, 1.0f };		// Zero scale not supported, return the identity
				else if (trace > 0.0f)
				{
					const float inv_trace = fp.inv_sqrt(fp.add(trace, 1.0f));
					const float half_inv_trace = fp.mul(inv_trace, 0.5f);
					q.x = fp.mul(fp.sub(m[1][2], m[2][1]), half_inv_trace);
					q.y = fp.mul(fp.sub(m[2][0], m[0][2]), half_inv_trace);
					q.z = fp.mul(fp.sub(m[0][1], m[1][0]), half_inv_trace);
					q.w = fp.mul(__fdiv_rn(1.0f, inv_trace), 0.5f);
					q = quat_normalize(fp, q);
				}
				else
				{
					// best axis = the largest diagonal element; the three cases are the reference's index arithmetic written out
					const int best = m[2][2] > (m[1][1] > m[0][0] ? m[1][1] : m[0][0]) ? 2 : (m[1][1] > m[0][0] ? 1 : 0);
					float d_best, d_next, d_next_next, s_next, s_next_next, s_w;
					if (best == 0)		{ d_best = m[0][0]; d_next = m[1][1]; d_next_next = m[2][2]; s_next = fp.add(m[0][1], m[1][0]); s_next_next = fp.add(m[0][2], m[2][0]); s_w = fp.sub(m[1][2], m[2][1]); }
					else if (best == 1)	{ d_best = m[1][1]; d_next = m[2][2]; d_next_next = m[0][0]; s_next = fp.add(m[1][2], m[2][1]); s_next_next = fp.add(m[1][0], m[0][1]); s_w = fp.sub(m[2][0], m[0][2]); }
					else				{ d_best = m[2][2]; d_next = m[0][0]; d_next_next = m[1][1]; s_next = fp.add(m[2][0], m[0][2]); s_next_next = fp.add(m[2][1], m[1][2]); s_w = fp.sub(m[0][1], m[1][0]); }
					const float pseudo_trace = fp.sub(fp.sub(fp.add(1.0f, d_best), d_next), d_next_next);
					const float inv_pseudo_trace = fp.inv_sqrt(pseudo_trace);
					const float half_inv_pseudo_trace = fp.mul(inv_pseudo_trace, 0.5f);
					const float v_best = fp.mul(__fdiv_rn(1.0f, inv_pseudo_trace), 0.5f);
					const float v_next = fp.mul(half_inv_pseudo_trace, s_next);
					const float v_next_next = fp.mul(half_inv_pseudo_trace, s_next_next);
					q.w = fp.mul(half_inv_pseudo_trace, s_w);
					if (best == 0)		{ q.x = v_best; q.y = v_next; q.z = v_next_next; }
					else if (best == 1)	{ q.y = v_best; q.z = v_next; q.x = v_next_next; }
					else				{ q.z = v_best; q.x = v_next; q.y = v_next_next; }
					q = quat_normalize(fp, q);
				}
				Qvv<float> result;
				result.rotation = q;
				result.translation = Vec3<float>{ m[3][0], m[3][1], m[3][2] };
				result.scale = Vec3<float>{ scale[0], scale[1], scale[2] };
				*out = result;
			}

			// rtm::qvv_mul(lhs, rhs), external/rtm/includes/rtm/qvvf.h:315-355, the positive scale branch (:347-353)
			template<class V>
			__device__ __forceinline__ Qvv<V> qvv_mul_positive(const Fp<V>& fp, const Qvv<V>& lhs, const Qvv<V>& rhs)
			{
				Qvv<V> out;
				out.rotation = quat_mul(fp, lhs.rotation, rhs.rotation);
				Vec3<V> scaled;
				scaled.x = fp.mul(lhs.translation.x, rhs.scale.x);
				scaled.y = fp.mul(lhs.translation.y, rhs.scale.y);
				scaled.z = fp.mul(lhs.translation.z, rhs.scale.z);
				const Vec3<V> rotated = quat_mul_vector3(fp, scaled, rhs.rotation);
				out.translation.x = fp.add(rotated.x, rhs.translation.x);
				out.translation.y = fp.add(rotated.y, rhs.translation.y);
				out.translation.z = fp.add(rotated.z, rhs.translation.z);
				out.scale.x = fp.mul(lhs.scale.x, rhs.scale.x);
				out.scale.y = fp.mul(lhs.scale.y, rhs.scale.y);
				out.scale.z = fp.mul(lhs.scale.z, rhs.scale.z);
				return out;
			}

			// which branch rtm::qvv_mul takes: vector_any_less_than3(vector_min(lhs.scale, rhs.scale), 0), qvvf.h:317-320 (either stream of a pair)
			template<class V>
			__device__ __forceinline__ bool takes_negative_branch(const Fp<V>& fp, const Vec3<V>& lhs_scale, const Vec3<V>& rhs_scale)
			{
				return fp.any_negative(lhs_scale.x, rhs_scale.x) || fp.any_negative(lhs_scale.y, rhs_scale.y) || fp.any_negative(lhs_scale.z, rhs_scale.z);
			}

			// acl::apply_additive_to_base(format, base, additive), includes/acl/core/additive_utils.h:131-167 (format = additive_clip_format8:
			// 1 relative = qvv_mul(additive, base), 2 additive0, 3 additive1; transform_add0 / transform_add1 :131-145), positive scales.
			// Format 0 (none) is the caller's business: it returns the additive transform unchanged.
			template<class V>
			__device__ __forceinline__ Qvv<V> apply_additive_to_base_positive(const Fp<V>& fp, uint32_t format, const Qvv<V>& base, const Qvv<V>& additive)
			{
				if (format == 1)
					return qvv_mul_positive(fp, additive, base);
				Qvv<V> out;
				out.rotation = quat_mul(fp, additive.rotation, base.rotation);
				out.translation.x = fp.add(additive.translation.x, base.translation.x);
				out.translation.y = fp.add(additive.translation.y, base.translation.y);
				out.translation.z = fp.add(additive.translation.z, base.translation.z);
				if (format == 2)
				{
					out.scale.x = fp.mul(additive.scale.x, base.scale.x);
					out.scale.y = fp.mul(additive.scale.y, base.scale.y);
					out.scale.z = fp.mul(additive.scale.z, base.scale.z);
				}
				else
				{
					const V one = fp.splat(1.0f);
					out.scale.x = fp.mul(fp.add(one, additive.scale.x), base.scale.x);
					out.scale.y = fp.mul(fp.add(one, additive.scale.y), base.scale.y);
					out.scale.z = fp.mul(fp.add(one, additive.scale.z), base.scale.z);
				}
				return out;
			}

			// ---- qvvf_matrix3x4f_transform_error_metric (transform_error_metrics.h:389-464): the same walk on 3x4 matrices. Every operation is an
			// IEEE mul / add / sqrt: this metric is bit-identical to the reference on any CPU ----
			template<class V> struct Mat34 { V m[4][3]; };		// rows: x_axis, y_axis, z_axis, w_axis (translation)

			// rtm::matrix_from_qvv, matrix3x4f.h:134-159 (convert_transforms :397-413)
			template<class V>
			__device__ __forceinline__ Mat34<V> matrix_from_qvv(const Fp<V>& fp, const Qvv<V>& q)
			{
				const V x2 = fp.add(q.rotation.x, q.rotation.x), y2 = fp.add(q.rotation.y, q.rotation.y), z2 = fp.add(q.rotation.z, q.rotation.z);
				const V xx = fp.mul(q.rotation.x, x2), xy = fp.mul(q.rotation.x, y2), xz = fp.mul(q.rotation.x, z2);
				const V yy = fp.mul(q.rotation.y, y2), yz = fp.mul(q.rotation.y, z2), zz = fp.mul(q.rotation.z, z2);
				const V wx = fp.mul(q.rotation.w, x2), wy = fp.mul(q.rotation.w, y2), wz = fp.mul(q.rotation.w, z2);
				const V one = fp.splat(1.0f);
				Mat34<V> out;
				out.m[0][0] = fp.mul(fp.sub(one, fp.add(yy, zz)), q.scale.x);	out.m[0][1] = fp.mul(fp.add(xy, wz), q.scale.x);				out.m[0][2] = fp.mul(fp.sub(xz, wy), q.scale.x);
				out.m[1][0] = fp.mul(fp.sub(xy, wz), q.scale.y);				out.m[1][1] = fp.mul(fp.sub(one, fp.add(xx, zz)), q.scale.y);	out.m[1][2] = fp.mul(fp.add(yz, wx), q.scale.y);
				out.m[2][0] = fp.mul(fp.add(xz, wy), q.scale.z);				out.m[2][1] = fp.mul(fp.sub(yz, wx), q.scale.z);				out.m[2][2] = fp.mul(fp.sub(one, fp.add(xx, yy)), q.scale.z);
				out.m[3][0] = q.translation.x;									out.m[3][1] = q.translation.y;									out.m[3][2] = q.translation.z;
				return out;
			}

			// rtm::matrix_mul(lhs, rhs), matrix3x4f.h:298-321 (local_to_object_space :415-436)
			template<class V>
			__device__ __forceinline__ Mat34<V> matrix_mul(const Fp<V>& fp, const Mat34<V>& l, const Mat34<V>& r)
			{
				Mat34<V> out;
				#pragma unroll
				for (int row = 0; row < 4; ++row)
					#pragma unroll
					for (int c = 0; c < 3; ++c)
					{
						V tmp = fp.mul(l.m[row][0], r.m[0][c]);
						tmp = fp.add(fp.mul(l.m[row][1], r.m[1][c]), tmp);
						tmp = fp.add(fp.mul(l.m[row][2], r.m[2][c]), tmp);
						out.m[row][c] = row == 3 ? fp.add(r.m[3][c], tmp) : tmp;
					}
				return out;
			}

			template<class V>
			__device__ __forceinline__ void store_matrix_planes(V* planes, uint32_t plane_stride, uint32_t bone, const Mat34<V>& q)
			{
				#pragma unroll
				for (int row = 0; row < 4; ++row)
					#pragma unroll
					for (int c = 0; c < 3; ++c)
						planes[(row * 3 + c) * plane_stride + bone] = q.m[row][c];
			}

			template<class V>
			__device__ __forceinline__ Mat34<V> load_matrix_planes(const V* planes, uint32_t plane_stride, uint32_t bone)
			{
				Mat34<V> q;
				#pragma unroll
				for (int row = 0; row < 4; ++row)
					#pragma unroll
					for (int c = 0; c < 3; ++c)
						q.m[row][c] = planes[(row * 3 + c) * plane_stride + bone];
				return q;
			}

			// object transforms of a warp's pose in shared memory: [component][bone] planes of V (32 lanes reading 32 different parents hit
			// different banks; a float2 plane element is one 8 byte access)
			template<class V>
			__device__ __forceinline__ void store_planes(V* planes, uint32_t plane_stride, uint32_t bone, const Qvv<V>& q)
			{
				planes[0 * plane_stride + bone] = q.rotation.x;
				planes[1 * plane_stride + bone] = q.rotation.y;
				planes[2 * plane_stride + bone] = q.rotation.z;
				planes[3 * plane_stride + bone] = q.rotation.w;
				planes[4 * plane_stride + bone] = q.translation.x;
				planes[5 * plane_stride + bone] = q.translation.y;
				planes[6 * plane_stride + bone] = q.translation.z;
				planes[7 * plane_stride + bone] = q.scale.x;
				planes[8 * plane_stride + bone] = q.scale.y;
				planes[9 * plane_stride + bone] = q.scale.z;
			}

			template<class V>
			__device__ __forceinline__ Qvv<V> load_planes(const V* planes, uint32_t plane_stride, uint32_t bone)
			{
				Qvv<V> q;
				q.rotation.x = planes[0 * plane_stride + bone];
				q.rotation.y = planes[1 * plane_stride + bone];
				q.rotation.z = planes[2 * plane_stride + bone];
				q.rotation.w = planes[3 * plane_stride + bone];
				q.translation.x = planes[4 * plane_stride + bone];
				q.translation.y = planes[5 * plane_stride + bone];
				q.translation.z = planes[6 * plane_stride + bone];
				q.scale.x = planes[7 * plane_stride + bone];
				q.scale.y = planes[8 * plane_stride + bone];
				q.scale.z = planes[9 * plane_stride + bone];
				return q;
			}

			// ---- the out of line paths: a bone whose qvv_mul takes the negative scale branch in either stream. They work on the planes in
			// shared memory, stream by stream on plain floats, so that the packed registers of the fast path never meet a conditional
			// assignment (a packed value that is conditionally modified gets split into its halves and re-paired with moves) ----
			template<class V> struct Streams;
			template<> struct Streams<float> { static constexpr int count = 1; };
			template<> struct Streams<float2> { static constexpr int count = 2; };

			template<class V>
			__device__ __forceinline__ Qvv<float> read_stream(const V* planes, uint32_t plane_stride, uint32_t bone, int stream)
			{
				const float* words = reinterpret_cast<const float*>(planes);
				const auto at = [&](uint32_t component) { return words[(size_t(component) * plane_stride + bone) * Streams<V>::count + stream]; };
				Qvv<float> q;
				q.rotation = Quat<float>{ at(0), at(1), at(2), at(3) };
				q.translation = Vec3<float>{ at(4), at(5), at(6) };
				q.scale = Vec3<float>{ at(7), at(8), at(9) };
				return q;
			}

			template<class V>
			__device__ __forceinline__ void write_stream(V* planes, uint32_t plane_stride, uint32_t bone, int stream, const Qvv<float>& q)
			{
				float* words = reinterpret_cast<float*>(planes);
				const auto put = [&](uint32_t component, float value) { words[(size_t(component) * plane_stride + bone) * Streams<V>::count + stream] = value; };
				put(0, q.rotation.x); put(1, q.rotation.y); put(2, q.rotation.z); put(3, q.rotation.w);
				put(4, q.translation.x); put(5, q.translation.y); put(6, q.translation.z);
				put(7, q.scale.x); put(8, q.scale.y); put(9, q.scale.z);
			}

			// rtm::qvv_mul on one stream, whichever branch it takes
			__device__ __forceinline__ Qvv<float> qvv_mul_any(const Qvv<float>& lhs, const Qvv<float>& rhs)
			{
				const Fp<float> fp{};
				if (!takes_negative_branch(fp, lhs.scale, rhs.scale))
					return qvv_mul_positive(fp, lhs, rhs);
				Qvv<float> out;
				qvv_mul_negative_scale(&lhs, &rhs, &out);
				return out;
			}

			// rtm::qvv_inverse(input), qvvf.h:389-395, the one argument form (root motion, root_motion.cu): quat_conjugate (the sign bits of x, y
			// and z xor-ed, quatf.h:482-491), vector_reciprocal as the IEEE division 1 / scale (_mm_div_ps, vector4f.h:1310), then
			// -quat_mul_vector3(translation * inv_scale, inv_rotation) with vector_neg's sign xor (vector4f.h:1261-1271). No normalisation.
			__device__ __forceinline__ Qvv<float> qvv_inverse(const Qvv<float>& input)
			{
				const Fp<float> fp{};
				const auto neg = [](float v) { return __uint_as_float(__float_as_uint(v) ^ 0x80000000u); };
				Qvv<float> out;
				out.rotation = Quat<float>{ neg(input.rotation.x), neg(input.rotation.y), neg(input.rotation.z), input.rotation.w };
				out.scale = Vec3<float>{ __fdiv_rn(1.0f, input.scale.x), __fdiv_rn(1.0f, input.scale.y), __fdiv_rn(1.0f, input.scale.z) };
				const Vec3<float> scaled = { fp.mul(input.translation.x, out.scale.x), fp.mul(input.translation.y, out.scale.y),
					fp.mul(input.translation.z, out.scale.z) };
				const Vec3<float> rotated = quat_mul_vector3(fp, scaled, out.rotation);
				out.translation = Vec3<float>{ neg(rotated.x), neg(rotated.y), neg(rotated.z) };
				return out;
			}

			// rtm::qvv_mul(lhs, rhs) through whichever branch it takes; the matrix branch (a mirrored operand) is reported
			__device__ __forceinline__ Qvv<float> flagged_qvv_mul(const Qvv<float>& lhs, const Qvv<float>& rhs, uint32_t& flags)
			{
				if (takes_negative_branch(Fp<float>{}, lhs.scale, rhs.scale))
					flags |= ACLB200_ERROR_FLAG_NEGATIVE_SCALE;
				return qvv_mul_any(lhs, rhs);
			}

			// M of aclb200_extract_root_motion from the root samples T(from), T(to), T(D) (end) and T(0) (start), |cycles| <= 256: root
			// motion (root_motion.cu) composes it per request, the pose features (features.cu) per (request, offset). `clip_flags` is the
			// clip's ClipDesc::flags: a loop crossing on a clip compressed with the wrap policy is reported.
			__device__ __forceinline__ Qvv<float> compose_root_motion(const Qvv<float>& from, const Qvv<float>& to, const Qvv<float>& end,
				const Qvv<float>& start, int32_t cycles, uint32_t clip_flags, uint32_t& flags)
			{
				Qvv<float> motion;
				if (cycles == 0)
					motion = flagged_qvv_mul(to, qvv_inverse(from), flags);		// rel(from, to)
				else
				{
					// forward: the boundary reached is the end, playback resumes at the start; backward the other way round
					const bool forward = cycles > 0;
					const Qvv<float> reached = forward ? end : start;
					const Qvv<float> inverse_resumed = qvv_inverse(forward ? start : end);
					motion = flagged_qvv_mul(reached, qvv_inverse(from), flags);				// rel(from, reached)
					const Qvv<float> cycle = flagged_qvv_mul(reached, inverse_resumed, flags);		// rel(resumed, reached), once
					const int32_t full_cycles = (forward ? cycles : -cycles) - 1;
					for (int32_t i = 0; i < full_cycles; ++i)
						motion = flagged_qvv_mul(cycle, motion, flags);
					motion = flagged_qvv_mul(flagged_qvv_mul(to, inverse_resumed, flags), motion, flags);	// rel(resumed, to)
					if (clip_flags & k_clip_wrap)
						flags |= ACLB200_ERROR_FLAG_WRAP_CLIP_CYCLE;
				}
				return motion;
			}

			// planes[bone] = qvv_normalize(qvv_mul(planes[bone] (the local transform), planes[parent])), every stream
			template<class V>
			__device__ __noinline__ void object_transform_slow(V* planes, uint32_t plane_stride, uint32_t bone, uint32_t parent)
			{
				const Fp<float> fp{};
				for (int stream = 0; stream < Streams<V>::count; ++stream)
				{
					Qvv<float> out = qvv_mul_any(read_stream(planes, plane_stride, bone, stream), read_stream(planes, plane_stride, parent, stream));
					out.rotation = quat_normalize(fp, out.rotation);
					write_stream(planes, plane_stride, bone, stream, out);
				}
			}

			// A parent that does not precede its child: the reference would read an object transform it has not written yet. Reported, and
			// the bone is treated as a root.
			__device__ __forceinline__ bool parent_follows(bool active, uint32_t bone, uint32_t parent)
			{
				return active && parent != k_invalid_track && parent >= bone;
			}

			// The hierarchy walk of one chunk of 32 bones (bone = base + lane), in wavefronts: `compute()` runs on a lane once its parent's
			// object transform is final. Every lane of the warp calls it; roots and inactive lanes never compute.
			template<class Compute>
			__device__ __forceinline__ void wavefront_walk(bool active, uint32_t parent, uint32_t base, Compute&& compute)
			{
				bool pending = active && parent != k_invalid_track;
				uint32_t done_mask = __ballot_sync(0xFFFFFFFFu, active && !pending);
				while (__any_sync(0xFFFFFFFFu, pending))
				{
					const bool ready = pending && (parent < base || ((done_mask >> (parent - base)) & 1u) != 0);
					if (ready)
					{
						compute();
						pending = false;
					}
					__syncwarp();
					done_mask |= __ballot_sync(0xFFFFFFFFu, ready);
				}
			}

			// ---- the walk on 48 byte pose rows in shared memory (the object space decode): a bone's row holds its local rtm::qvvf (rotation
			// xyzw, translation xyz + 0, scale xyz + 0) and is overwritten in place by its object transform, as a qvvf row of the same layout
			// or as the xyz lanes of the matrix's x_axis, y_axis, z_axis, w_axis. A lane moves its own row with three 16 byte accesses: rows
			// are 48 bytes apart, so the 8 lanes of each quarter warp cover the 32 banks exactly once (no conflict) ----
			__device__ __forceinline__ Qvv<float> load_qvv_row(const float4* row)
			{
				const float4 r = row[0], t = row[1], s = row[2];
				Qvv<float> q;
				q.rotation = Quat<float>{ r.x, r.y, r.z, r.w };
				q.translation = Vec3<float>{ t.x, t.y, t.z };
				q.scale = Vec3<float>{ s.x, s.y, s.z };
				return q;
			}

			__device__ __forceinline__ void store_qvv_row(float4* row, const Qvv<float>& q)
			{
				row[0] = make_float4(q.rotation.x, q.rotation.y, q.rotation.z, q.rotation.w);
				row[1] = make_float4(q.translation.x, q.translation.y, q.translation.z, 0.0f);
				row[2] = make_float4(q.scale.x, q.scale.y, q.scale.z, 0.0f);
			}

			__device__ __forceinline__ Mat34<float> load_matrix_row(const float4* row)
			{
				const float4 a = row[0], b = row[1], c = row[2];
				return Mat34<float>{ { { a.x, a.y, a.z }, { a.w, b.x, b.y }, { b.z, b.w, c.x }, { c.y, c.z, c.w } } };
			}

			__device__ __forceinline__ void store_matrix_row(float4* row, const Mat34<float>& m)
			{
				row[0] = make_float4(m.m[0][0], m.m[0][1], m.m[0][2], m.m[1][0]);
				row[1] = make_float4(m.m[1][1], m.m[1][2], m.m[2][0], m.m[2][1]);
				row[2] = make_float4(m.m[2][2], m.m[3][0], m.m[3][1], m.m[3][2]);
			}

			// row = qvv_normalize(qvv_mul(row (the local transform), parent_row)) through whichever branch qvv_mul takes
			__device__ __noinline__ void object_row_slow(float4* row, const float4* parent_row)
			{
				const Fp<float> fp{};
				Qvv<float> out = qvv_mul_any(load_qvv_row(row), load_qvv_row(parent_row));
				out.rotation = quat_normalize(fp, out.rotation);
				store_qvv_row(row, out);
			}

			// One warp takes the pose at `pose` (num_tracks rows of 48 bytes in shared memory) to object space with the skeleton `parents`:
			// qvvf_transform_error_metric::local_to_object_space (transform_error_metrics.h:289-310) or, MATRIX, convert_transforms +
			// local_to_object_space of qvvf_matrix3x4f_transform_error_metric (:397-436). Every lane of the warp calls it; returns the lane's
			// ACLB200_ERROR_FLAG_* bits.
			// CLOSURE (the bone query): only the bones of `closure` (bit b % 32 of word b / 32: bone b; no bit at or above num_tracks), an
			// ancestor-closed set: the parent of a closure bone is in the closure, unless it does not precede the bone (then the bone is a
			// root, as in the whole walk). The same row operations and wavefronts on the closure bones only, chunks of 32 bones without one
			// skipped: a closure row ends byte for byte as the whole walk leaves it, and no other row is read or written. A template
			// argument rather than a run-time mask, so that the whole walk's code carries no mask.
			template<bool CLOSURE = false>
			__device__ __forceinline__ uint32_t pose_rows_to_object_space(uint8_t* pose, uint32_t num_tracks, const uint32_t* parents, bool matrix,
				const uint32_t* closure = nullptr)
			{
				const Fp<float> fp{};
				const uint32_t lane = threadIdx.x & 31u;
				uint32_t flags = 0;
				for (uint32_t base = 0; base < num_tracks; base += 32)
				{
					uint32_t word = 0;
					if (CLOSURE)
					{
						word = closure[base >> 5];
						if (word == 0)
							continue;
					}
					const uint32_t bone = base + lane;
					const bool active = CLOSURE ? ((word >> lane) & 1u) != 0 : bone < num_tracks;
					uint32_t parent = active ? __ldg(parents + bone) : k_invalid_track;
					if (parent_follows(active, bone, parent))
					{
						flags |= ACLB200_ERROR_FLAG_INVALID_SKELETON;
						parent = k_invalid_track;
					}
					float4* row = reinterpret_cast<float4*>(pose + size_t(bone) * 48);
					if (matrix)
					{
						if (active)
							store_matrix_row(row, matrix_from_qvv(fp, load_qvv_row(row)));		// convert_transforms
						__syncwarp();
						wavefront_walk(active, parent, base, [&]()
						{
							const float4* above = reinterpret_cast<const float4*>(pose + size_t(parent) * 48);
							store_matrix_row(row, matrix_mul(fp, load_matrix_row(row), load_matrix_row(above)));
						});
					}
					else
					{
						wavefront_walk(active, parent, base, [&]()
						{
							const float4* above = reinterpret_cast<const float4*>(pose + size_t(parent) * 48);
							const Qvv<float> mine = load_qvv_row(row);
							const Qvv<float> up = load_qvv_row(above);
							if (takes_negative_branch(fp, mine.scale, up.scale))
							{
								flags |= ACLB200_ERROR_FLAG_NEGATIVE_SCALE;
								object_row_slow(row, above);
							}
							else
							{
								// rtm::qvv_normalize(rtm::qvv_mul(local, parent_object)), qvvf.h:426-430
								Qvv<float> object = qvv_mul_positive(fp, mine, up);
								object.rotation = quat_normalize(fp, object.rotation);
								store_qvv_row(row, object);
							}
						});
					}
				}
				return flags;
			}

			// ---- the skinning step (the skinning decodes and aclb200_local_to_skinning): after pose_rows_to_object_space(..., matrix = true)
			// has walked the WHOLE pose, row b becomes rtm::matrix_mul(inverse_bind[b], object[b]) (rtm's row vector order: a bind pose
			// vertex goes into the bone's space, then on to the model). It must not start earlier: a child in a later chunk of 32 bones
			// reads its parent's object matrix from that row. The inverse binds are the 12 float layout of the matrix rows (x_axis, y_axis,
			// z_axis, w_axis, xyz each), 16 byte aligned; the result leaves as three float4 rows of the skinning matrix's transpose, row c =
			// (x_axis[c], y_axis[c], z_axis[c], w_axis[c]), so that dot(row c, (p, 1)) is component c of rtm::matrix_mul_point3(p, skin).
			// Every lane of the warp calls it; a lane only touches the rows of its own bones ----
			__device__ __forceinline__ void skin_pose_rows(uint8_t* pose, uint32_t num_tracks, const float* inverse_bind)
			{
				const Fp<float> fp{};
				__syncwarp();
				for (uint32_t bone = threadIdx.x & 31u; bone < num_tracks; bone += 32)
				{
					float4* row = reinterpret_cast<float4*>(pose + size_t(bone) * 48);
					const float4* bind = reinterpret_cast<const float4*>(inverse_bind + size_t(bone) * 12);
					const float4 a = __ldg(bind), b = __ldg(bind + 1), c = __ldg(bind + 2);
					const Mat34<float> inverse = { { { a.x, a.y, a.z }, { a.w, b.x, b.y }, { b.z, b.w, c.x }, { c.y, c.z, c.w } } };
					const Mat34<float> skin = matrix_mul(fp, inverse, load_matrix_row(row));
					row[0] = make_float4(skin.m[0][0], skin.m[1][0], skin.m[2][0], skin.m[3][0]);
					row[1] = make_float4(skin.m[0][1], skin.m[1][1], skin.m[2][1], skin.m[3][1]);
					row[2] = make_float4(skin.m[0][2], skin.m[1][2], skin.m[2][2], skin.m[3][2]);
				}
			}

			// ---- apply_additive_to_base on pose rows (the additive decode and aclb200_apply_additive_to_base): one thread per bone, a row of 48
			// bytes (QVV48: rotation xyzw, translation xyz + 0, scale xyz + 0, 16 byte aligned) or 40 bytes (QVV40: rotation xyzw, translation
			// xyz, scale xyz, 8 byte aligned) ----
			__device__ __forceinline__ Qvv<float> load_pose_row(const uint8_t* row, bool qvv40)
			{
				if (!qvv40)
					return load_qvv_row(reinterpret_cast<const float4*>(row));
				const float2* r = reinterpret_cast<const float2*>(row);
				const float2 a = r[0], b = r[1], c = r[2], d = r[3], e = r[4];
				Qvv<float> q;
				q.rotation = Quat<float>{ a.x, a.y, b.x, b.y };
				q.translation = Vec3<float>{ c.x, c.y, d.x };
				q.scale = Vec3<float>{ d.y, e.x, e.y };
				return q;
			}

			__device__ __forceinline__ void store_pose_row(uint8_t* row, const Qvv<float>& q, bool qvv40)
			{
				if (!qvv40)
				{
					store_qvv_row(reinterpret_cast<float4*>(row), q);
					return;
				}
				float2* r = reinterpret_cast<float2*>(row);
				r[0] = make_float2(q.rotation.x, q.rotation.y);
				r[1] = make_float2(q.rotation.z, q.rotation.w);
				r[2] = make_float2(q.translation.x, q.translation.y);
				r[3] = make_float2(q.translation.z, q.scale.x);
				r[4] = make_float2(q.scale.y, q.scale.z);
			}

			// out_row = rtm::qvv_mul(additive_row, base_row) through the matrix branch (a mirrored bone of a `relative` clip)
			__device__ __noinline__ void additive_relative_row_slow(uint8_t* out_row, const uint8_t* base_row, const uint8_t* additive_row, bool qvv40)
			{
				const Qvv<float> base = load_pose_row(base_row, qvv40);
				const Qvv<float> additive = load_pose_row(additive_row, qvv40);
				Qvv<float> out;
				qvv_mul_negative_scale(&additive, &base, &out);
				store_pose_row(out_row, out, qvv40);
			}

			// out_row = acl::apply_additive_to_base(format, base_row, additive_row) (additive_utils.h:152-162; format 0 = none, the additive
			// row itself). out_row may be either input. Returns ACLB200_ERROR_FLAG_NEGATIVE_SCALE when `relative` took qvv_mul's matrix branch.
			__device__ __forceinline__ uint32_t apply_additive_row(uint8_t* out_row, const uint8_t* base_row, const uint8_t* additive_row, uint32_t format,
				bool qvv40)
			{
				const Fp<float> fp{};
				const Qvv<float> base = load_pose_row(base_row, qvv40);
				const Qvv<float> additive = load_pose_row(additive_row, qvv40);
				if (format == 1 && takes_negative_branch(fp, additive.scale, base.scale))
				{
					additive_relative_row_slow(out_row, base_row, additive_row, qvv40);
					return ACLB200_ERROR_FLAG_NEGATIVE_SCALE;
				}
				store_pose_row(out_row, format == 0 ? additive : apply_additive_to_base_positive(fp, format, base, additive), qvv40);
				return 0;
			}

			// rtm::vector_lerp, vector4f.h:2417-2421 with the SSE2 macros (macros.vector4.impl.h:93,152): (start - start * alpha) + end * alpha
			__device__ __forceinline__ float lerp_lane(const Fp<float>& fp, float start, float end, float alpha)
			{
				return fp.add(fp.sub(start, fp.mul(start, alpha)), fp.mul(end, alpha));
			}

			// out_row = rtm::qvv_lerp(from_row, to_row, weight) (qvvf.h:439-445), rows as apply_additive_row's; out_row may be either input.
			// quat_lerp is its SSE4.1 path (quatf.h:1006-1075): dot = _mm_dp_ps(start, end, 0xFF), which sums (x x' + y y') + (z z' + w w');
			// the SIGN BIT of dot is xor-ed onto `end` (so dot == -0.0 flips it, unlike the scalar and NEON paths); (s - w s) + w (e ^ bias) per
			// lane, then quat_normalize with the IEEE 1 / sqrt in place of rsqrtss + 2 Newton-Raphson steps. The weight is used as given: no
			// clamp, below 0 and above 1 extrapolate.
			__device__ __forceinline__ void blend_row(uint8_t* out_row, const uint8_t* from_row, const uint8_t* to_row, float weight, bool qvv40)
			{
				const Fp<float> fp{};
				const Qvv<float> from = load_pose_row(from_row, qvv40);
				const Qvv<float> to = load_pose_row(to_row, qvv40);
				const Quat<float>& s = from.rotation;
				const Quat<float>& e = to.rotation;
				const float dot = fp.add(fp.add(fp.mul(s.x, e.x), fp.mul(s.y, e.y)), fp.add(fp.mul(s.z, e.z), fp.mul(s.w, e.w)));
				const uint32_t bias = __float_as_uint(dot) & 0x80000000u;
				const auto biased = [bias](float v) { return __uint_as_float(__float_as_uint(v) ^ bias); };
				Quat<float> q;
				q.x = fp.add(fp.sub(s.x, fp.mul(weight, s.x)), fp.mul(weight, biased(e.x)));
				q.y = fp.add(fp.sub(s.y, fp.mul(weight, s.y)), fp.mul(weight, biased(e.y)));
				q.z = fp.add(fp.sub(s.z, fp.mul(weight, s.z)), fp.mul(weight, biased(e.z)));
				q.w = fp.add(fp.sub(s.w, fp.mul(weight, s.w)), fp.mul(weight, biased(e.w)));
				Qvv<float> out;
				out.rotation = quat_normalize(fp, q);
				out.translation = Vec3<float>{ lerp_lane(fp, from.translation.x, to.translation.x, weight), lerp_lane(fp, from.translation.y, to.translation.y, weight),
					lerp_lane(fp, from.translation.z, to.translation.z, weight) };
				out.scale = Vec3<float>{ lerp_lane(fp, from.scale.x, to.scale.x, weight), lerp_lane(fp, from.scale.y, to.scale.y, weight),
					lerp_lane(fp, from.scale.z, to.scale.z, weight) };
				store_pose_row(out_row, out, qvv40);
			}

			// ---- inertialization (aclb200_begin_inertialization, aclb200_inertialize_poses): rtm's quat_rotation_log and quat_rotation_exp
			// (quatf.h:1306-1375) on their SSE2 paths, which are polynomials and IEEE operations only, so they match the reference on any CPU.
			// rtm's float constants are static_cast<float> of its double literals (constants.h:35-47) ----
			constexpr float k_rtm_pi = float(3.141592653589793238462643383279502884);
			constexpr float k_rtm_half_pi = float(1.570796326794896619231321691639751442);
			constexpr float k_rtm_two_pi = float(6.283185307179586476925286766559005768);
			constexpr float k_rtm_one_div_two_pi = float(1.591549430918953357688837633725143620e-01);

			// rtm::scalar_acos, scalarf.h:1142-1174: a degree 7 polynomial in |v| times sqrt(1 - |v|), reflected for v < 0
			__device__ __forceinline__ float rtm_acos(float v)
			{
				const Fp<float> fp{};
				const float x = fabsf(v);
				float r = fp.add(fp.mul(x, -1.2690614339589956e-3f), 6.7072304676685235e-3f);
				r = fp.sub(fp.mul(r, x), 1.7162031184398074e-2f);
				r = fp.add(fp.mul(r, x), 3.0961594977611639e-2f);
				r = fp.sub(fp.mul(r, x), 5.0207843052845647e-2f);
				r = fp.add(fp.mul(r, x), 8.8986946573346160e-2f);
				r = fp.sub(fp.mul(r, x), 2.1459960076929829e-1f);
				r = fp.add(fp.mul(r, x), 1.5707963267948966f);
				r = fp.mul(r, __fsqrt_rn(fp.sub(1.0f, x)));
				return v < 0.0f ? fp.sub(k_rtm_pi, r) : r;
			}

			// the range reduction of rtm::scalar_sin and scalar_cos (scalarf.h:855-967): angle - bankers_round(angle / 2 pi) * 2 pi (roundss
			// under SSE4.1, rint here), then reflected about copysign(pi, x) when |x| > pi / 2 (the compare is false for NaN)
			__device__ __forceinline__ float rtm_reduce_angle(float angle, bool& within_half_pi)
			{
				const Fp<float> fp{};
				const float x = fp.sub(angle, fp.mul(rintf(fp.mul(angle, k_rtm_one_div_two_pi)), k_rtm_two_pi));
				within_half_pi = fabsf(x) <= k_rtm_half_pi;
				return within_half_pi ? x : fp.sub(copysignf(k_rtm_pi, x), x);
			}

			// rtm::scalar_sin (SSE2 path): a degree 11 polynomial
			__device__ __forceinline__ float rtm_sin(float angle)
			{
				const Fp<float> fp{};
				bool within_half_pi;
				const float x = rtm_reduce_angle(angle, within_half_pi);
				const float x2 = fp.mul(x, x);
				float r = fp.add(fp.mul(x2, -2.3828544692960918e-8f), 2.7521557770526783e-6f);
				r = fp.sub(fp.mul(r, x2), 1.9840782426250314e-4f);
				r = fp.add(fp.mul(r, x2), 8.3333303183525942e-3f);
				r = fp.sub(fp.mul(r, x2), 1.6666666601721269e-1f);
				r = fp.add(fp.mul(r, x2), 1.0f);
				return fp.mul(r, x);
			}

			// rtm::scalar_cos (SSE2 path): a degree 10 polynomial whose sign bit is set (OR-ed, not flipped) when the angle was reflected
			__device__ __forceinline__ float rtm_cos(float angle)
			{
				const Fp<float> fp{};
				bool within_half_pi;
				const float x = rtm_reduce_angle(angle, within_half_pi);
				const float x2 = fp.mul(x, x);
				float r = fp.add(fp.mul(x2, -2.6051615464872668e-7f), 2.4760495088926859e-5f);
				r = fp.sub(fp.mul(r, x2), 1.3888377661039897e-3f);
				r = fp.add(fp.mul(r, x2), 4.1666638865338612e-2f);
				r = fp.sub(fp.mul(r, x2), 4.9999999508695869e-1f);
				r = fp.add(fp.mul(r, x2), 1.0f);
				return within_half_pi ? r : __uint_as_float(__float_as_uint(r) | 0x80000000u);
			}

			// rtm::quat_rotation_log(q).xyz (its w is 0): w clamped to [-1, 1] by _mm_min_ss(_mm_max_ss(w, -1), 1) (NaN becomes -1),
			// xyz * ((1 / sqrt((x x + y y) + z z)) * acos(w)), or xyz itself when the clamped w > 1 - 1e-6
			__device__ __forceinline__ Vec3<float> quat_rotation_log(const Quat<float>& q)
			{
				const Fp<float> fp{};
				const float lower = q.w > -1.0f ? q.w : -1.0f;
				const float w = lower < 1.0f ? lower : 1.0f;
				const float half_angle = rtm_acos(w);
				const float inv_len = fp.inv_sqrt(fp.add(fp.add(fp.mul(q.x, q.x), fp.mul(q.y, q.y)), fp.mul(q.z, q.z)));
				const float s = fp.mul(inv_len, half_angle);
				if (w > 1.0f - 1.0e-6f)
					return Vec3<float>{ q.x, q.y, q.z };
				return Vec3<float>{ fp.mul(q.x, s), fp.mul(q.y, s), fp.mul(q.z, s) };
			}

			// rtm::quat_rotation_exp((v, w)): len = sqrt((x x + y y) + z z), xyz = (v / len) * sin(len), or v itself when len < 1e-6;
			// w = cos(len)
			__device__ __forceinline__ Quat<float> quat_rotation_exp(const Vec3<float>& v)
			{
				const Fp<float> fp{};
				const float len = __fsqrt_rn(fp.add(fp.add(fp.mul(v.x, v.x), fp.mul(v.y, v.y)), fp.mul(v.z, v.z)));
				const float sine = rtm_sin(len);
				Quat<float> out;
				out.w = rtm_cos(len);
				if (len < 1.0e-6f)
				{
					out.x = v.x; out.y = v.y; out.z = v.z;
				}
				else
				{
					out.x = fp.mul(__fdiv_rn(v.x, len), sine);
					out.y = fp.mul(__fdiv_rn(v.y, len), sine);
					out.z = fp.mul(__fdiv_rn(v.z, len), sine);
				}
				return out;
			}

			// 2 log(abs(rtm::quat_mul(conj(from), to))).xyz: the scaled angle axis of the rotation that takes `from` to `to` (Hamilton
			// to from^-1). abs negates all four lanes when w < 0 (an IEEE compare: -0 stays); conj flips the sign bits of x, y and z.
			__device__ __forceinline__ Vec3<float> scaled_angle_axis_between(const Quat<float>& from, const Quat<float>& to)
			{
				const Fp<float> fp{};
				const Quat<float> conj{ -from.x, -from.y, -from.z, from.w };
				Quat<float> q = quat_mul(fp, conj, to);
				if (q.w < 0.0f)
					q = Quat<float>{ -q.x, -q.y, -q.z, -q.w };
				const Vec3<float> l = quat_rotation_log(q);
				return Vec3<float>{ fp.mul(2.0f, l.x), fp.mul(2.0f, l.y), fp.mul(2.0f, l.z) };
			}

			// One bone's inertialization record entry from its displayed (src) and destination (dst) local rows this frame and the frame
			// before: rot_x, rot_v, pos_x, pos_v as four float4 (xyz, w = 0) at `entry`, 16 byte aligned. Velocities are backward differences
			// times inv_dt: (2 log(abs(quat_mul(conj(p_prev), p)))) * inv_dt and (t - t_prev) * inv_dt.
			__device__ __forceinline__ void capture_inertialization_row(float4* entry, const float4* src_row, const float4* src_prev_row,
				const float4* dst_row, const float4* dst_prev_row, float inv_dt)
			{
				const Fp<float> fp{};
				const Qvv<float> src = load_qvv_row(src_row), src_prev = load_qvv_row(src_prev_row);
				const Qvv<float> dst = load_qvv_row(dst_row), dst_prev = load_qvv_row(dst_prev_row);
				const Vec3<float> rot_x = scaled_angle_axis_between(dst.rotation, src.rotation);
				const Vec3<float> src_w = scaled_angle_axis_between(src_prev.rotation, src.rotation);
				const Vec3<float> dst_w = scaled_angle_axis_between(dst_prev.rotation, dst.rotation);
				entry[0] = make_float4(rot_x.x, rot_x.y, rot_x.z, 0.0f);
				entry[1] = make_float4(fp.sub(fp.mul(src_w.x, inv_dt), fp.mul(dst_w.x, inv_dt)), fp.sub(fp.mul(src_w.y, inv_dt), fp.mul(dst_w.y, inv_dt)),
					fp.sub(fp.mul(src_w.z, inv_dt), fp.mul(dst_w.z, inv_dt)), 0.0f);
				entry[2] = make_float4(fp.sub(src.translation.x, dst.translation.x), fp.sub(src.translation.y, dst.translation.y),
					fp.sub(src.translation.z, dst.translation.z), 0.0f);
				const auto velocity = [&](float t, float t_prev) { return fp.mul(fp.sub(t, t_prev), inv_dt); };
				entry[3] = make_float4(fp.sub(velocity(src.translation.x, src_prev.translation.x), velocity(dst.translation.x, dst_prev.translation.x)),
					fp.sub(velocity(src.translation.y, src_prev.translation.y), velocity(dst.translation.y, dst_prev.translation.y)),
					fp.sub(velocity(src.translation.z, src_prev.translation.z), velocity(dst.translation.z, dst_prev.translation.z)), 0.0f);
			}

			// The critically damped spring of one request, from `elapsed` and `halflife` as given: y = (4 ln 2 / (halflife + 1e-5)) / 2,
			// e = fast_negexp(y elapsed) = 1 / (((1 + u) + (0.48 u) u) + ((0.235 u) u) u)
			struct InertializationDecay { float y, e, elapsed; };

			__device__ __forceinline__ InertializationDecay inertialization_decay(float elapsed, float halflife)
			{
				const Fp<float> fp{};
				InertializationDecay d;
				d.y = fp.mul(__fdiv_rn(2.7725887f, fp.add(halflife, 1.0e-5f)), 0.5f);
				const float u = fp.mul(d.y, elapsed);
				d.e = __fdiv_rn(1.0f, fp.add(fp.add(fp.add(1.0f, u), fp.mul(fp.mul(0.48f, u), u)), fp.mul(fp.mul(fp.mul(0.235f, u), u), u)));
				d.elapsed = elapsed;
				return d;
			}

			// x(x0, v0) = e (x0 + (v0 + x0 y) elapsed)
			__device__ __forceinline__ float decayed(const InertializationDecay& d, float x0, float v0)
			{
				const Fp<float> fp{};
				return fp.mul(d.e, fp.add(x0, fp.mul(fp.add(v0, fp.mul(x0, d.y)), d.elapsed)));
			}

			// out_row = the destination row `row` with its record entry's offset decayed onto it: rotation quat_mul(dst.q, exp(x(rot_x, rot_v)
			// * 0.5)) (Hamilton offset dst), translation dst.t + x(pos_x, pos_v), scale dst.s. Rows as apply_additive_row's (QVV48 or
			// QVV40); out_row may be row.
			__device__ __forceinline__ void inertialize_row(uint8_t* out_row, const uint8_t* row, const float4* entry, const InertializationDecay& d,
				bool qvv40)
			{
				const Fp<float> fp{};
				const float4 rot_x = entry[0], rot_v = entry[1], pos_x = entry[2], pos_v = entry[3];
				const Qvv<float> dst = load_pose_row(row, qvv40);
				const Vec3<float> half_offset{ fp.mul(decayed(d, rot_x.x, rot_v.x), 0.5f), fp.mul(decayed(d, rot_x.y, rot_v.y), 0.5f),
					fp.mul(decayed(d, rot_x.z, rot_v.z), 0.5f) };
				Qvv<float> out;
				out.rotation = quat_mul(fp, dst.rotation, quat_rotation_exp(half_offset));
				out.translation = Vec3<float>{ fp.add(dst.translation.x, decayed(d, pos_x.x, pos_v.x)), fp.add(dst.translation.y, decayed(d, pos_x.y, pos_v.y)),
					fp.add(dst.translation.z, decayed(d, pos_x.z, pos_v.z)) };
				out.scale = dst.scale;
				store_pose_row(out_row, out, qvv40);
			}

			// ---- mirroring (aclb200_mirror_poses, the mirrored decode): reflect_q flips the sign bits of the quaternion lanes other than
			// `axis`, reflect_t the translation lane `axis`; sign bit flips, so -0 / +0 swap and NaN payloads stay ----
			__device__ __forceinline__ float flip_sign(float v, bool flip)
			{
				return __uint_as_float(__float_as_uint(v) ^ (flip ? 0x80000000u : 0u));
			}

			// row i's partner among n rows: m = table[i].mirror when m < n and table[m].mirror == i, else i itself with invalid set
			__device__ __forceinline__ uint32_t mirror_partner(const aclb200_mirror_entry* table, uint32_t i, uint32_t n, bool& invalid)
			{
				const uint32_t m = __ldg(&table[i].mirror);
				if (m < n && __ldg(&table[m].mirror) == i)
					return m;
				invalid = true;
				return i;
			}

			// the mirrored row from the partner's row `src` and this row's entry: rotation quat_mul(quat_mul(pre, reflect_q(q)), post),
			// translation quat_mul_vector3(reflect_t(t), post), scale copied
			__device__ __forceinline__ Qvv<float> mirrored_row(const Qvv<float>& src, const aclb200_mirror_entry* entry, uint32_t axis)
			{
				const Fp<float> fp{};
				const float4 pre = __ldg(reinterpret_cast<const float4*>(entry->pre));
				const float4 post = __ldg(reinterpret_cast<const float4*>(entry->post));
				const Quat<float> reflected{ flip_sign(src.rotation.x, axis != 0), flip_sign(src.rotation.y, axis != 1),
					flip_sign(src.rotation.z, axis != 2), src.rotation.w };
				const Quat<float> post_q{ post.x, post.y, post.z, post.w };
				Qvv<float> out;
				out.rotation = quat_mul(fp, quat_mul(fp, Quat<float>{ pre.x, pre.y, pre.z, pre.w }, reflected), post_q);
				out.translation = quat_mul_vector3(fp, Vec3<float>{ flip_sign(src.translation.x, axis == 0), flip_sign(src.translation.y, axis == 1),
					flip_sign(src.translation.z, axis == 2) }, post_q);
				out.scale = src.scale;
				return out;
			}

			// A partner pair (row i, row m; the same row for a self partner) read from in_i / in_m and written to out_i / out_m, each from
			// the other's transform. Rows as apply_additive_row's (QVV48 or QVV40); the outputs may be the inputs.
			__device__ __forceinline__ void mirror_row(uint8_t* out_i, uint8_t* out_m, const uint8_t* in_i, const uint8_t* in_m,
				const aclb200_mirror_entry* entry_i, const aclb200_mirror_entry* entry_m, uint32_t axis, bool qvv40)
			{
				const Qvv<float> row_i = load_pose_row(in_i, qvv40);
				const Qvv<float> row_m = load_pose_row(in_m, qvv40);
				store_pose_row(out_i, mirrored_row(row_m, entry_i, axis), qvv40);
				if (entry_m != entry_i)
					store_pose_row(out_m, mirrored_row(row_i, entry_m, axis), qvv40);
			}
		}
	}
}
