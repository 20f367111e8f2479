// include/acl_b200/decompress.h -- C++ header shim over the C ABI of libaclb200 (include/aclb200.h).
//
// It keeps the reference's decompression front end (includes/acl/decompression/decompress.h:76-209) so that a call site switches
// by changing a namespace:
//
//   acl::decompression_context<my_settings> context;              acl_b200::decompression_context<my_settings> context;
//   context.initialize(*compressed_tracks);                       context.initialize(*compressed_tracks);
//   context.seek(sample_time, acl::sample_rounding_policy::none); context.seek(sample_time, acl::sample_rounding_policy::none);
//   context.decompress_tracks(writer);                            context.decompress_tracks(writer);
//   context.decompress_track(bone_index, writer);                 context.decompress_track(bone_index, writer);
//
// Two front ends, one implementation:
//   * the reference's headers are on the include path (-I<acl>/includes -I<rtm>/includes; detected with __has_include, or forced
//     with -DACLB200_WITH_ACL_HEADERS=1): the shim USES the reference's own types -- acl::compressed_tracks, acl::sample_rounding_policy,
//     acl::sample_looping_policy, any settings struct derived from acl::decompression_settings (static_assert as in decompress.h:197), any
//     writer derived from acl::track_writer with its rtm::quatf_arg0 / rtm::vector4f_arg0 / rtm::scalarf_arg0 arguments
//     (core/track_writer.h:82-216), e.g. acl::acl_impl::debug_track_writer. tests/cpp/shim_reference_callsite.cpp is the body of the
//     reference's own benchmark loop (tools/acl_decompressor/sources/benchmark.cpp:246-258) compiled against both classes.
//   * without them (-DACLB200_WITH_ACL_HEADERS=0): stand-alone mirrors of those types with the same member names live in
//     namespace acl_b200 (float4 instead of the rtm types).
//
// Semantics kept (decompress.impl.h:66-260): initialize() returns false for an invalid / unsupported buffer, for a track type,
// version or rotation / translation / scale format the settings do not support (a clip bound to a streaming database is accepted and
// decodes from its resident key frames, like a reference context initialised without its database; initialize(tracks, database_context)
// binds it to a database_context below, and it then decodes from the tiers streamed in); relocated() and
// is_bound_to() compare the hash (decompression.transform.h:134-176); seek() on an unbound context and decompress_*() before a
// seek() do nothing; transform AND scalar clips (write_float1..4 / write_vector4); every sample_rounding_policy including per_track
// (writer.get_rounding_policy per track); all default sub-track modes; skip_all_* / skip_track_*.
//
// A decompression_context decodes ONE pose per call through the GPU: a launch plus a PCIe round trip. It exists for drop-in
// compatibility and for tests. Throughput comes from batch_context / batch_decompressor below: upload the clips once, decode
// thousands of (clip, sample_time) requests per launch into device memory.
//
// Nothing here decodes on the CPU: without the library or without an H100 every call fails with a status, never silently.
#pragma once

#include "../aclb200.h"

#if !defined(ACLB200_WITH_ACL_HEADERS)
	#if defined(__has_include)
		#if __has_include(<acl/decompression/decompress.h>) && __has_include(<rtm/quatf.h>)
			#define ACLB200_WITH_ACL_HEADERS 1
		#endif
	#endif
	#if !defined(ACLB200_WITH_ACL_HEADERS)
		#define ACLB200_WITH_ACL_HEADERS 0
	#endif
#endif

#if ACLB200_WITH_ACL_HEADERS
	#include <acl/core/compressed_tracks.h>
	#include <acl/core/track_writer.h>
	#include <acl/decompression/decompression_settings.h>
	#include <acl/decompression/database/database.h>
	#include <rtm/quatf.h>
	#include <rtm/vector4f.h>
	#include <rtm/scalarf.h>
#endif

#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

namespace acl_b200
{
#if ACLB200_WITH_ACL_HEADERS
	// the reference's own vocabulary
	using acl::sample_rounding_policy;
	using acl::sample_looping_policy;
	using acl::rotation_normalization_policy_t;
	using acl::default_sub_track_mode;
	using acl::decompression_settings;
	using acl::default_transform_decompression_settings;
	using acl::debug_transform_decompression_settings;
	using acl::default_scalar_decompression_settings;
	using acl::debug_scalar_decompression_settings;
	using acl::track_writer;
	using acl::compressed_tracks;
	using acl::compressed_database;
	using acl::quality_tier;
	using acl::database_stream_request_result;
	using acl::default_database_settings;
#else
	// acl::sample_rounding_policy (core/sample_rounding_policy.h:47-107)
	enum class sample_rounding_policy : uint32_t { none = ACLB200_ROUND_NONE, floor = ACLB200_ROUND_FLOOR, ceil = ACLB200_ROUND_CEIL, nearest = ACLB200_ROUND_NEAREST, per_track = ACLB200_ROUND_PER_TRACK };
	// acl::sample_looping_policy (core/sample_looping_policy.h:56-82)
	enum class sample_looping_policy : uint32_t { clamp = ACLB200_LOOP_CLAMP, wrap = ACLB200_LOOP_WRAP, as_compressed = ACLB200_LOOP_AS_COMPRESSED };
	// acl::rotation_normalization_policy_t (decompression/decompression_settings.h:52-62)
	enum class rotation_normalization_policy_t : uint32_t { never = ACLB200_NORMALIZE_NEVER, lerp_only = ACLB200_NORMALIZE_LERP_ONLY, always = ACLB200_NORMALIZE_ALWAYS };
	// acl::default_sub_track_mode (core/track_writer.h:49-74)
	enum class default_sub_track_mode : uint32_t { skipped = ACLB200_DEFAULT_SKIPPED, constant = ACLB200_DEFAULT_CONSTANT, variable = ACLB200_DEFAULT_VARIABLE, legacy = ACLB200_DEFAULT_LEGACY };

	// What a writer receives: four floats (rotations xyzw; translations / scales xyz, w unspecified like in the reference)
	struct float4
	{
		float x, y, z, w;
	};

	// A view of a compressed_tracks buffer (core/compressed_tracks.h:53-203): the accessors the shim needs
	class compressed_tracks
	{
	public:
		uint32_t get_size() const { return read32(0); }
		uint32_t get_hash() const { return read32(4); }
		uint16_t get_version() const { uint16_t v; std::memcpy(&v, bytes() + 12, 2); return v; }
		uint8_t get_track_type() const { return bytes()[15]; }
		uint32_t get_num_tracks() const { return read32(16); }
	private:
		compressed_tracks() = delete;
		const uint8_t* bytes() const { return reinterpret_cast<const uint8_t*>(this); }
		uint32_t read32(size_t offset) const { uint32_t v; std::memcpy(&v, bytes() + offset, 4); return v; }
	};
	inline const compressed_tracks* make_compressed_tracks(const void* buffer) { return static_cast<const compressed_tracks*>(buffer); }

	// acl::compressed_database (core/compressed_database.h), acl::quality_tier (core/quality_tier.h), acl::database_stream_request_result
	// (decompression/database/database.h:48-73) and acl::default_database_settings (database_settings.h:79-84), same names and values
	class compressed_database
	{
	public:
		uint32_t get_size() const { uint32_t v; std::memcpy(&v, this, 4); return v; }
		uint32_t get_hash() const { uint32_t v; std::memcpy(&v, reinterpret_cast<const uint8_t*>(this) + 4, 4); return v; }
	private:
		compressed_database() = delete;
	};
	enum class quality_tier { highest_importance = 0, medium_importance = ACLB200_TIER_MEDIUM, lowest_importance = ACLB200_TIER_LOW };
	enum class database_stream_request_result { done, dispatched, streaming_in_progress, context_not_initialized, invalid_database_tier, no_free_streaming_requests };
	struct default_database_settings {};

	// acl::decompression_settings (decompression_settings.h:74-166), same member names and defaults
	struct decompression_settings
	{
		static constexpr bool clamp_sample_time() { return true; }
		static constexpr bool is_track_type_supported(uint32_t /*ACLB200_TRACK_**/) { return true; }
		static constexpr uint32_t version_supported() { return 0; }		// compressed_tracks_version16::any
		static constexpr bool is_rotation_format_supported(uint32_t /*rotation_format8*/) { return true; }
		static constexpr bool is_translation_format_supported(uint32_t /*vector_format8*/) { return true; }
		static constexpr bool is_scale_format_supported(uint32_t /*vector_format8*/) { return true; }
		static constexpr rotation_normalization_policy_t get_rotation_normalization_policy() { return rotation_normalization_policy_t::always; }
		static constexpr bool skip_initialize_safety_checks() { return false; }
		static constexpr bool is_wrapping_supported() { return true; }
		static constexpr bool is_per_track_rounding_supported() { return true; }
	};
	using debug_transform_decompression_settings = decompression_settings;		// decompression_settings.h:172-176
	using debug_scalar_decompression_settings = decompression_settings;
	// acl::default_transform_decompression_settings (decompression_settings.h:211-232)
	struct default_transform_decompression_settings : decompression_settings
	{
		static constexpr bool is_track_type_supported(uint32_t type) { return type == ACLB200_TRACK_QVVF; }
		static constexpr bool is_rotation_format_supported(uint32_t format) { return format == 3; }		// quatf_drop_w_variable
		static constexpr bool is_translation_format_supported(uint32_t format) { return format == 1; }	// vector3f_variable
		static constexpr bool is_scale_format_supported(uint32_t format) { return format == 1; }
		static constexpr rotation_normalization_policy_t get_rotation_normalization_policy() { return rotation_normalization_policy_t::lerp_only; }
		static constexpr bool is_per_track_rounding_supported() { return false; }
	};
	// acl::default_scalar_decompression_settings (decompression_settings.h:183-199)
	struct default_scalar_decompression_settings : decompression_settings
	{
		static constexpr bool is_track_type_supported(uint32_t type) { return type != ACLB200_TRACK_QVVF; }
		static constexpr bool is_per_track_rounding_supported() { return false; }
	};

	// acl::track_writer (core/track_writer.h:82-216), same member names and defaults
	struct track_writer
	{
		sample_rounding_policy get_rounding_policy(sample_rounding_policy seek_policy, uint32_t /*track_index*/) const { return seek_policy; }
		bool skip_track_float1(uint32_t) const { return false; }
		bool skip_track_float2(uint32_t) const { return false; }
		bool skip_track_float3(uint32_t) const { return false; }
		bool skip_track_float4(uint32_t) const { return false; }
		bool skip_track_vector4(uint32_t) const { return false; }
		void write_float1(uint32_t, float) {}
		void write_float2(uint32_t, float4) {}
		void write_float3(uint32_t, float4) {}
		void write_float4(uint32_t, float4) {}
		void write_vector4(uint32_t, float4) {}
		static constexpr default_sub_track_mode get_default_rotation_mode() { return default_sub_track_mode::constant; }
		static constexpr default_sub_track_mode get_default_translation_mode() { return default_sub_track_mode::constant; }
		static constexpr default_sub_track_mode get_default_scale_mode() { return default_sub_track_mode::legacy; }
		float4 get_constant_default_rotation() const { return float4{ 0.0F, 0.0F, 0.0F, 1.0F }; }
		float4 get_constant_default_translation() const { return float4{ 0.0F, 0.0F, 0.0F, 0.0F }; }
		float4 get_constant_default_scale() const { return float4{ 1.0F, 1.0F, 1.0F, 1.0F }; }
		float4 get_variable_default_rotation(uint32_t) const { return float4{ 0.0F, 0.0F, 0.0F, 1.0F }; }
		float4 get_variable_default_translation(uint32_t) const { return float4{ 0.0F, 0.0F, 0.0F, 0.0F }; }
		float4 get_variable_default_scale(uint32_t) const { return float4{ 1.0F, 1.0F, 1.0F, 1.0F }; }
		static constexpr bool skip_all_rotations() { return false; }
		static constexpr bool skip_all_translations() { return false; }
		static constexpr bool skip_all_scales() { return false; }
		bool skip_track_rotation(uint32_t) const { return false; }
		bool skip_track_translation(uint32_t) const { return false; }
		bool skip_track_scale(uint32_t) const { return false; }
		void write_rotation(uint32_t, float4) {}
		void write_translation(uint32_t, float4) {}
		void write_scale(uint32_t, float4) {}
	};
#endif

	class error : public std::runtime_error
	{
	public:
		error(aclb200_status status_, const std::string& what_) : std::runtime_error(what_), status(status_) {}
		aclb200_status status;
	};

	// One CUDA device. Owns the library context.
	class device_context
	{
	public:
		explicit device_context(int device = 0)
		{
			const aclb200_status status = aclb200_create(device, &m_context);
			if (status != ACLB200_OK)
				throw error(status, std::string("aclb200_create: ") + aclb200_status_string(status));
		}
		~device_context() { aclb200_destroy(m_context); }
		device_context(const device_context&) = delete;
		device_context& operator=(const device_context&) = delete;

		aclb200_context* get() const { return m_context; }
		void check(aclb200_status status, const char* what) const
		{
			if (status != ACLB200_OK)
				throw error(status, std::string(what) + ": " + aclb200_last_error(m_context));
		}

		// What a default constructed decompression_context uses: device 0, created on first use, shared by the thread's contexts
		// (an aclb200_context is single-owner state, like a reference context)
		static device_context& default_device()
		{
			thread_local device_context device(0);
			return device;
		}

	private:
		aclb200_context* m_context = nullptr;
	};

	namespace shim_impl
	{
		// ---- the two front ends differ only in these conversions ----
#if ACLB200_WITH_ACL_HEADERS
		inline rtm::quatf make_rotation(const float* p) { return rtm::quat_load(p); }
		inline rtm::vector4f make_vector(const float* p) { return rtm::vector_load(p); }
		inline rtm::scalarf make_scalar(const float* p) { return rtm::scalar_set(*p); }
		inline void store(rtm::quatf_arg0 q, float* out) { rtm::quat_store(q, out); }
		inline void store_vector(rtm::vector4f_arg0 v, float* out) { rtm::vector_store(v, out); }
		inline uint32_t version_number(acl::compressed_tracks_version16 version) { return static_cast<uint32_t>(version); }
		inline uint32_t track_type_number(acl::track_type8 type) { return static_cast<uint32_t>(type); }
		template<class settings> inline bool supports_track_type(uint32_t type) { return settings::is_track_type_supported(static_cast<acl::track_type8>(type)); }
		template<class settings> inline bool supports_rotation_format(uint32_t format) { return settings::is_rotation_format_supported(static_cast<acl::rotation_format8>(format)); }
		template<class settings> inline bool supports_translation_format(uint32_t format) { return settings::is_translation_format_supported(static_cast<acl::vector_format8>(format)); }
		template<class settings> inline bool supports_scale_format(uint32_t format) { return settings::is_scale_format_supported(static_cast<acl::vector_format8>(format)); }
#else
		inline float4 make_rotation(const float* p) { return float4{ p[0], p[1], p[2], p[3] }; }
		inline float4 make_vector(const float* p) { return float4{ p[0], p[1], p[2], p[3] }; }
		inline float make_scalar(const float* p) { return *p; }
		inline void store(float4 q, float* out) { out[0] = q.x; out[1] = q.y; out[2] = q.z; out[3] = q.w; }
		inline void store_vector(float4 v, float* out) { out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w; }
		inline uint32_t version_number(uint32_t version) { return version; }
		inline uint32_t track_type_number(uint32_t type) { return type; }
		template<class settings> inline bool supports_track_type(uint32_t type) { return settings::is_track_type_supported(type); }
		template<class settings> inline bool supports_rotation_format(uint32_t format) { return settings::is_rotation_format_supported(format); }
		template<class settings> inline bool supports_translation_format(uint32_t format) { return settings::is_translation_format_supported(format); }
		template<class settings> inline bool supports_scale_format(uint32_t format) { return settings::is_scale_format_supported(format); }
#endif

		// more than one rotation format compiled in (debug settings): changes the result for quatf_full clips sampled exactly on a
		// key frame (decompression_context.transform.h:191-200)
		template<class settings> inline bool supports_multiple_rotation_formats()
		{
			return int(supports_rotation_format<settings>(0)) + int(supports_rotation_format<settings>(2)) + int(supports_rotation_format<settings>(3)) > 1;
		}

		inline uint32_t read_u32(const void* base, size_t offset)
		{
			uint32_t v;
			std::memcpy(&v, static_cast<const uint8_t*>(base) + offset, 4);
			return v;
		}

		// a device allocation of the library (the shim never links the CUDA runtime)
		class device_buffer
		{
		public:
			device_buffer() = default;
			device_buffer(const device_buffer&) = delete;
			device_buffer& operator=(const device_buffer&) = delete;
			~device_buffer() { release(); }
			void* get(device_context& device, size_t bytes)
			{
				if (bytes > m_bytes || m_device != &device)
				{
					release();
					device.check(aclb200_device_malloc(device.get(), bytes, &m_pointer), "aclb200_device_malloc");
					m_bytes = bytes;
					m_device = &device;
				}
				return m_pointer;
			}
			void release()
			{
				if (m_pointer != nullptr)
					aclb200_device_free(m_device->get(), m_pointer);
				m_pointer = nullptr;
				m_bytes = 0;
			}
		private:
			device_context* m_device = nullptr;
			void* m_pointer = nullptr;
			size_t m_bytes = 0;
		};
	}

	template<class settings_type, class writer_type>
	inline aclb200_options make_options(const writer_type& writer, sample_rounding_policy rounding, sample_looping_policy looping)
	{
		aclb200_options options;
		std::memset(&options, 0, sizeof(options));
		aclb200_default_options(&options);
		options.rounding_policy = static_cast<uint32_t>(rounding);
		options.looping_policy = static_cast<uint32_t>(looping);
		options.normalization = static_cast<uint32_t>(settings_type::get_rotation_normalization_policy());
		options.per_track_rounding = settings_type::is_per_track_rounding_supported() ? 1u : 0u;
		options.wrapping = settings_type::is_wrapping_supported() ? 1u : 0u;
		options.clamp_sample_time = settings_type::clamp_sample_time() ? 1u : 0u;
		options.multiple_rotation_formats = shim_impl::supports_multiple_rotation_formats<settings_type>() ? 1u : 0u;
		// `variable` defaults come from writer callbacks: the device leaves those sub-tracks alone (skipped) and the replay asks the
		// writer, which is exactly what the reference does (decompression.transform.h:1566-1650)
		const auto device_mode = [](default_sub_track_mode mode) { return static_cast<uint32_t>(mode == default_sub_track_mode::variable ? default_sub_track_mode::skipped : mode); };
		options.default_rotation_mode = device_mode(writer_type::get_default_rotation_mode());
		options.default_translation_mode = device_mode(writer_type::get_default_translation_mode());
		options.default_scale_mode = device_mode(writer_type::get_default_scale_mode());
		float defaults[12] = {};
		shim_impl::store(writer.get_constant_default_rotation(), defaults);
		shim_impl::store_vector(writer.get_constant_default_translation(), defaults + 4);
		shim_impl::store_vector(writer.get_constant_default_scale(), defaults + 8);
		defaults[7] = defaults[11] = 0.0F;
		std::memcpy(options.constant_defaults, defaults, sizeof(defaults));
		options.output_layout = ACLB200_LAYOUT_QVV48;
		return options;
	}

	// The throughput interface: a set of clips resident in HBM + batched decodes into device memory.
	// Replaces N x { context.initialize(clip); context.seek(t, policy); context.decompress_tracks(writer); } by ONE launch.
	class batch_decompressor
	{
	public:
		explicit batch_decompressor(device_context& device) : m_device(&device) {}
		~batch_decompressor() { release(); }
		batch_decompressor(const batch_decompressor&) = delete;
		batch_decompressor& operator=(const batch_decompressor&) = delete;

		// compressed_tracks buffers as the reference's compressor wrote them (16 byte alignment not required here).
		// Returns false and reports the offending clip when one is not a valid / supported compressed_tracks instance,
		// which is what decompression_context::initialize() reports by returning false.
		bool upload(const void* const* blobs, const uint32_t* sizes, uint32_t num_clips, bool check_hash = true, uint32_t* out_failed_clip = nullptr)
		{
			release();
			const aclb200_status status = aclb200_upload_clips(m_device->get(), blobs, sizes, num_clips, check_hash ? 1u : 0u, &m_clipset, out_failed_clip);
			if (status == ACLB200_ERR_INVALID_CLIP || status == ACLB200_ERR_UNSUPPORTED)
				return false;
			m_device->check(status, "aclb200_upload_clips");
			m_device->check(aclb200_clipset_get_info(m_clipset, &m_info), "aclb200_clipset_get_info");
			return true;
		}
		void release()
		{
			if (m_clipset != nullptr)
				aclb200_release_clipset(m_device->get(), m_clipset);
			m_clipset = nullptr;
		}

		// decompression_context::initialize(tracks, database) for the clips of the batch (NULL unbinds): false, and the offending clip, when
		// the database does not contain a clip bound to a database
		bool bind_database(const aclb200_database* database, uint32_t* out_failed_clip = nullptr)
		{
			const aclb200_status status = aclb200_clipset_bind_database(m_device->get(), m_clipset, database, out_failed_clip);
			if (status == ACLB200_ERR_INVALID_CLIP)
				return false;
			m_device->check(status, "aclb200_clipset_bind_database");
			return true;
		}

		device_context& device() const { return *m_device; }
		const aclb200_clipset_info& info() const { return m_info; }
		const aclb200_clipset* clipset() const { return m_clipset; }

		// d_requests / d_out are DEVICE pointers; `stream` a cudaStream_t. Asynchronous like any kernel launch.
		void decompress_tracks(const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options& options, void* d_out, void* stream = nullptr)
		{
			if (m_info.track_type == ACLB200_TRACK_QVVF)
				m_device->check(aclb200_decompress_tracks(m_device->get(), m_clipset, d_requests, num_requests, &options, d_out, stream), "aclb200_decompress_tracks");
			else
				m_device->check(aclb200_scalar_decompress_tracks(m_device->get(), m_clipset, d_requests, num_requests, &options, d_out, stream), "aclb200_scalar_decompress_tracks");
		}
		void decompress_track(const aclb200_request* d_requests, const uint32_t* d_track_indices, uint32_t num_requests, const aclb200_options& options, void* d_out, void* stream = nullptr)
		{
			if (m_info.track_type == ACLB200_TRACK_QVVF)
				m_device->check(aclb200_decompress_track(m_device->get(), m_clipset, d_requests, d_track_indices, num_requests, &options, d_out, stream), "aclb200_decompress_track");
			else
				m_device->check(aclb200_scalar_decompress_track(m_device->get(), m_clipset, d_requests, d_track_indices, num_requests, &options, d_out, stream), "aclb200_scalar_decompress_track");
		}
		// decompress_tracks() + the hierarchy walk in one launch (aclb200_decompress_tracks_object_space): object space bones of 48 bytes,
		// ACLB200_OBJECT_QVVF or ACLB200_OBJECT_MATRIX3X4F; clip c uses the skeleton at d_parent_indices + d_skeleton_offsets[c] (nullptr: 0)
		void decompress_tracks_object_space(const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options& options,
			const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, uint32_t object_kind, void* d_out, uint32_t* d_out_flags = nullptr,
			void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_object_space(m_device->get(), m_clipset, d_requests, num_requests, &options, d_parent_indices,
				d_skeleton_offsets, object_kind, d_out, d_out_flags, stream), "aclb200_decompress_tracks_object_space");
		}
		// decompress base + decompress additive (track_writer defaults) + acl::apply_additive_to_base per bone, in one launch
		// (aclb200_decompress_tracks_additive). Format: d_clip_additive_formats[additive clip] (nullptr: additive_format). With parents the
		// combined pose leaves in object space as object_kind rows (the base clip's skeleton), else as local rows in options.output_layout.
		void decompress_tracks_additive(const aclb200_additive_request* d_requests, uint32_t num_requests, const aclb200_options& options,
			uint32_t additive_format, const uint8_t* d_clip_additive_formats, void* d_out, const uint32_t* d_parent_indices = nullptr,
			const uint32_t* d_skeleton_offsets = nullptr, uint32_t object_kind = ACLB200_OBJECT_QVVF, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_additive(m_device->get(), m_clipset, d_requests, num_requests, &options, additive_format,
				d_clip_additive_formats, d_parent_indices, d_skeleton_offsets, object_kind, d_out, d_out_flags, stream), "aclb200_decompress_tracks_additive");
		}
		// acl::apply_additive_to_base over num_poses QVV48 poses already on the device (aclb200_apply_additive_to_base); d_out may be either input
		void apply_additive_to_base(const void* d_base_poses, const void* d_additive_poses, void* d_out, uint64_t num_poses, uint32_t num_tracks,
			uint32_t additive_format, uint64_t pose_stride_bytes = 0, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_apply_additive_to_base(m_device->get(), d_base_poses, d_additive_poses, d_out, num_poses, num_tracks, pose_stride_bytes,
				additive_format, d_out_flags, stream), "aclb200_apply_additive_to_base");
		}
		// decompress from + decompress to + rtm::qvv_lerp(from, to, w) per bone, in one launch (aclb200_decompress_tracks_blend); w =
		// d_weights[r] (nullptr: weight). With parents the blended pose leaves in object space as object_kind rows (the from clip's
		// skeleton), else as local rows in options.output_layout.
		void decompress_tracks_blend(const aclb200_blend_request* d_requests, uint32_t num_requests, const aclb200_options& options,
			float weight, const float* d_weights, void* d_out, const uint32_t* d_parent_indices = nullptr, const uint32_t* d_skeleton_offsets = nullptr,
			uint32_t object_kind = ACLB200_OBJECT_QVVF, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_blend(m_device->get(), m_clipset, d_requests, num_requests, &options, weight, d_weights,
				d_parent_indices, d_skeleton_offsets, object_kind, d_out, d_out_flags, stream), "aclb200_decompress_tracks_blend");
		}
		// rtm::qvv_lerp(from, to, w) over num_poses QVV48 poses already on the device (aclb200_blend_poses); d_out may be either input
		void blend_poses(const void* d_from_poses, const void* d_to_poses, void* d_out, uint64_t num_poses, uint32_t num_tracks, float weight,
			const float* d_weights = nullptr, uint64_t pose_stride_bytes = 0, void* stream = nullptr)
		{
			m_device->check(aclb200_blend_poses(m_device->get(), d_from_poses, d_to_poses, d_out, num_poses, num_tracks, pose_stride_bytes, weight,
				d_weights, stream), "aclb200_blend_poses");
		}
		// Up to eight layers per pose in one launch (aclb200_decompress_tracks_layered): pose r owns d_layers[r * num_layers + i]; the first
		// layer that is not ACLB200_LAYER_OFF is the base, decoded as decompress_tracks decodes it, and each later layer is folded in, in
		// order: BLEND = rtm::qvv_lerp(running, layer, weight), ADDITIVE = acl::apply_additive_to_base(format, running, layer) with the layer
		// decoded with the track_writer defaults, OFF = skipped unread. Format: d_clip_additive_formats[layer clip] (nullptr: additive_format).
		// With parents the running pose leaves in object space as object_kind rows (the base clip's skeleton), else as local rows in
		// options.output_layout.
		void decompress_tracks_layered(const aclb200_layer* d_layers, uint32_t num_poses, uint32_t num_layers, const aclb200_options& options,
			uint32_t additive_format, const uint8_t* d_clip_additive_formats, void* d_out, const uint32_t* d_parent_indices = nullptr,
			const uint32_t* d_skeleton_offsets = nullptr, uint32_t object_kind = ACLB200_OBJECT_QVVF, uint32_t* d_out_flags = nullptr,
			void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_layered(m_device->get(), m_clipset, d_layers, num_poses, num_layers, &options, additive_format,
				d_clip_additive_formats, d_parent_indices, d_skeleton_offsets, object_kind, d_out, d_out_flags, stream), "aclb200_decompress_tracks_layered");
		}
		// Skinning rows: the ACLB200_OBJECT_MATRIX3X4F walk, then rtm::matrix_mul(inverse_bind, object) per bone, stored as three float4 rows,
		// row c = (x_axis[c], y_axis[c], z_axis[c], w_axis[c]). d_inverse_bind holds 12 floats per skeleton entry, 16 byte aligned, in
		// parallel with d_parent_indices (aclb200_decompress_tracks_skinning and its additive, blend and standalone forms)
		void decompress_tracks_skinning(const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options& options,
			const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind, void* d_out,
			uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_skinning(m_device->get(), m_clipset, d_requests, num_requests, &options, d_parent_indices,
				d_skeleton_offsets, d_inverse_bind, d_out, d_out_flags, stream), "aclb200_decompress_tracks_skinning");
		}
		void decompress_tracks_additive_skinning(const aclb200_additive_request* d_requests, uint32_t num_requests, const aclb200_options& options,
			uint32_t additive_format, const uint8_t* d_clip_additive_formats, const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets,
			const float* d_inverse_bind, void* d_out, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_additive_skinning(m_device->get(), m_clipset, d_requests, num_requests, &options, additive_format,
				d_clip_additive_formats, d_parent_indices, d_skeleton_offsets, d_inverse_bind, d_out, d_out_flags, stream),
				"aclb200_decompress_tracks_additive_skinning");
		}
		void decompress_tracks_blend_skinning(const aclb200_blend_request* d_requests, uint32_t num_requests, const aclb200_options& options,
			float weight, const float* d_weights, const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets, const float* d_inverse_bind,
			void* d_out, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_blend_skinning(m_device->get(), m_clipset, d_requests, num_requests, &options, weight, d_weights,
				d_parent_indices, d_skeleton_offsets, d_inverse_bind, d_out, d_out_flags, stream), "aclb200_decompress_tracks_blend_skinning");
		}
		void decompress_tracks_layered_skinning(const aclb200_layer* d_layers, uint32_t num_poses, uint32_t num_layers, const aclb200_options& options,
			uint32_t additive_format, const uint8_t* d_clip_additive_formats, const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets,
			const float* d_inverse_bind, void* d_out, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_layered_skinning(m_device->get(), m_clipset, d_layers, num_poses, num_layers, &options,
				additive_format, d_clip_additive_formats, d_parent_indices, d_skeleton_offsets, d_inverse_bind, d_out, d_out_flags, stream),
				"aclb200_decompress_tracks_layered_skinning");
		}
		// Masked layer stacks (aclb200_decompress_tracks_layered_masked): decompress_tracks_layered where layer i of pose r may name a bone
		// mask d_layer_masks[r * num_layers + i] (ACLB200_LAYER_NO_MASK: none; d_layer_masks nullptr: no masks), mask m being
		// d_bone_masks[m * mask_stride + b] per bone b of the base clip (mask_stride 0: max_tracks). At bone b the layer's weight is
		// weight * mask[b], and a mask of +-0 leaves the bone untouched; ADDITIVE layers take their weight (the additive delta lerped from the
		// track_writer defaults when it is not 1). ADDITIVE weights 1 without masks give decompress_tracks_layered's bytes.
		void decompress_tracks_layered_masked(const aclb200_layer* d_layers, const uint32_t* d_layer_masks, uint32_t num_poses, uint32_t num_layers,
			const float* d_bone_masks, uint32_t num_masks, uint32_t mask_stride, const aclb200_options& options, uint32_t additive_format,
			const uint8_t* d_clip_additive_formats, void* d_out, const uint32_t* d_parent_indices = nullptr, const uint32_t* d_skeleton_offsets = nullptr,
			uint32_t object_kind = ACLB200_OBJECT_QVVF, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_layered_masked(m_device->get(), m_clipset, d_layers, d_layer_masks, num_poses, num_layers,
				d_bone_masks, num_masks, mask_stride, &options, additive_format, d_clip_additive_formats, d_parent_indices, d_skeleton_offsets,
				object_kind, d_out, d_out_flags, stream), "aclb200_decompress_tracks_layered_masked");
		}
		void decompress_tracks_layered_masked_skinning(const aclb200_layer* d_layers, const uint32_t* d_layer_masks, uint32_t num_poses,
			uint32_t num_layers, const float* d_bone_masks, uint32_t num_masks, uint32_t mask_stride, const aclb200_options& options,
			uint32_t additive_format, const uint8_t* d_clip_additive_formats, const uint32_t* d_parent_indices, const uint32_t* d_skeleton_offsets,
			const float* d_inverse_bind, void* d_out, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_layered_masked_skinning(m_device->get(), m_clipset, d_layers, d_layer_masks, num_poses,
				num_layers, d_bone_masks, num_masks, mask_stride, &options, additive_format, d_clip_additive_formats, d_parent_indices,
				d_skeleton_offsets, d_inverse_bind, d_out, d_out_flags, stream), "aclb200_decompress_tracks_layered_masked_skinning");
		}
		// Bone queries (aclb200_decompress_bones): entry j of request r's bone list (list d_request_lists[r], or list 0 when it is nullptr;
		// list l is d_bone_lists[l * bones_per_list ..], ACLB200_NO_BONE for a hole) lands at d_out + r * pose_stride + j * bone size. Without
		// parents, row list[j] of decompress_tracks; with them, row list[j] of decompress_tracks_object_space as object_kind rows. Only the
		// listed bones' ancestor chains are decoded and walked.
		void decompress_bones(const aclb200_request* d_requests, uint32_t num_requests, const aclb200_options& options, const uint32_t* d_bone_lists,
			uint32_t num_lists, uint32_t bones_per_list, void* d_out, const uint32_t* d_request_lists = nullptr, const uint32_t* d_parent_indices = nullptr,
			const uint32_t* d_skeleton_offsets = nullptr, uint32_t object_kind = ACLB200_OBJECT_QVVF, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_bones(m_device->get(), m_clipset, d_requests, num_requests, &options, d_bone_lists, num_lists, bones_per_list,
				d_request_lists, d_parent_indices, d_skeleton_offsets, object_kind, d_out, d_out_flags, stream), "aclb200_decompress_bones");
		}
		// Root motion (aclb200_extract_root_motion): the root's delta M between each request's from_time and to_time across `cycles` loop
		// boundaries, one 48 byte rtm::qvvf row per request at d_out + r * 48; the root of clip c is d_root_tracks[c] (nullptr: track 0).
		// options need the QVV48 layout and ACLB200_LOOP_CLAMP. An engine accumulates M as character = rtm::qvv_mul(M, character).
		void extract_root_motion(const aclb200_root_motion_request* d_requests, uint32_t num_requests, const aclb200_options& options, void* d_out,
			const uint32_t* d_root_tracks = nullptr, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_extract_root_motion(m_device->get(), m_clipset, d_requests, num_requests, &options, d_root_tracks, d_out, d_out_flags,
				stream), "aclb200_extract_root_motion");
		}
		// Pose features (aclb200_extract_pose_features): for each request and each of the num_offsets host `offsets` (seconds, 1..8), the
		// object rows of its bone list's bones at t + offset (wrapped into the clip for ACLB200_FEATURE_LOOP requests) in the root's frame at
		// t, row (s, k) of request r at d_out + r * pose_stride + (s * bones_per_list + k) * 48. The root of clip c is d_root_tracks[c]
		// (nullptr: track 0), its skeleton d_parent_indices + d_skeleton_offsets[c]. options need the QVV48 layout and ACLB200_LOOP_CLAMP.
		void extract_pose_features(const aclb200_feature_request* d_requests, uint32_t num_requests, const aclb200_options& options,
			const float* offsets, uint32_t num_offsets, const uint32_t* d_bone_lists, uint32_t num_lists, uint32_t bones_per_list,
			const uint32_t* d_parent_indices, void* d_out, const uint32_t* d_request_lists = nullptr, const uint32_t* d_root_tracks = nullptr,
			const uint32_t* d_skeleton_offsets = nullptr, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_extract_pose_features(m_device->get(), m_clipset, d_requests, num_requests, &options, offsets, num_offsets,
				d_bone_lists, num_lists, bones_per_list, d_request_lists, d_root_tracks, d_parent_indices, d_skeleton_offsets, d_out, d_out_flags,
				stream), "aclb200_extract_pose_features");
		}
		// Motion matching (aclb200_pack_pose_features): extract_pose_features rows of num_requests requests (S = num_offsets, K =
		// bones_per_list) into vectors of num_dims floats, out[r][d] = (v_d - mean[d]) * scale[d] at d_out + r * out_stride floats. `terms`,
		// `mean` and `scale` are host arrays (mean / scale nullptr: 0 / 1); pose_stride_bytes 0 = S * K rows.
		void pack_pose_features(const void* d_rows, uint32_t num_requests, uint32_t num_offsets, uint32_t bones_per_list,
			const aclb200_feature_term* terms, uint32_t num_terms, uint32_t num_dims, float* d_out, uint32_t out_stride, const float* mean = nullptr,
			const float* scale = nullptr, uint64_t pose_stride_bytes = 0, void* stream = nullptr)
		{
			m_device->check(aclb200_pack_pose_features(m_device->get(), d_rows, num_requests, num_offsets, bones_per_list, pose_stride_bytes, terms,
				num_terms, mean, scale, num_dims, d_out, out_stride, stream), "aclb200_pack_pose_features");
		}
		// Motion matching (aclb200_search_pose_features): the lowest cost allowed database row of each query (the lowest row on a tie,
		// {ACLB200_NO_ROW, +inf} without one); strides in floats, d_row_tags nullptr: every row allowed by every tag mask.
		void search_pose_features(const float* d_database, uint64_t num_rows, uint64_t db_stride, const float* d_query_vectors,
			const aclb200_search_query* d_queries, uint32_t num_queries, uint64_t q_stride, uint32_t num_dims, aclb200_search_result* d_results,
			const uint32_t* d_row_tags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_search_pose_features(m_device->get(), d_database, num_rows, db_stride, d_row_tags, d_query_vectors, d_queries,
				num_queries, q_stride, num_dims, d_results, stream), "aclb200_search_pose_features");
		}
		// The inertialization record of each transition (aclb200_begin_inertialization): from the displayed QVV48 poses this frame and the
		// frame before and the destination poses, one frame being 1 / inv_dt seconds; transition j writes record d_record_slots[j], or j.
		void begin_inertialization(const void* d_src, const void* d_src_prev, const void* d_dst, const void* d_dst_prev, uint64_t num_transitions,
			uint32_t num_tracks, float inv_dt, void* d_records, const uint32_t* d_record_slots = nullptr, uint64_t pose_stride_bytes = 0,
			uint64_t record_stride_bytes = 0, void* stream = nullptr)
		{
			m_device->check(aclb200_begin_inertialization(m_device->get(), d_src, d_src_prev, d_dst, d_dst_prev, num_transitions, num_tracks,
				pose_stride_bytes, inv_dt, d_records, record_stride_bytes, d_record_slots, stream), "aclb200_begin_inertialization");
		}
		// Each QVV48 pose with its record's offset decayed onto it (aclb200_inertialize_poses); d_out may be d_poses
		void inertialize_poses(const void* d_poses, void* d_out, uint64_t num_poses, uint32_t num_tracks,
			const aclb200_inertialization* d_inertializations, const void* d_records, uint64_t num_records, uint64_t pose_stride_bytes = 0,
			uint64_t record_stride_bytes = 0, void* stream = nullptr)
		{
			m_device->check(aclb200_inertialize_poses(m_device->get(), d_poses, d_out, num_poses, num_tracks, pose_stride_bytes, d_inertializations,
				d_records, num_records, record_stride_bytes, stream), "aclb200_inertialize_poses");
		}
		// Decode and inertialize in one launch (aclb200_decompress_tracks_inertialized): local rows without parents, object space rows of
		// `object_kind` with them; ACLB200_NO_INERTIALIZATION requests as the plain decodes write them
		void decompress_tracks_inertialized(const aclb200_inertialized_request* d_requests, uint32_t num_requests, const aclb200_options& options,
			const void* d_records, uint64_t num_records, void* d_out, uint64_t record_stride_bytes = 0, const uint32_t* d_parent_indices = nullptr,
			const uint32_t* d_skeleton_offsets = nullptr, uint32_t object_kind = ACLB200_OBJECT_QVVF, uint32_t* d_out_flags = nullptr,
			void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_inertialized(m_device->get(), m_clipset, d_requests, num_requests, &options, d_records,
				num_records, record_stride_bytes, d_parent_indices, d_skeleton_offsets, object_kind, d_out, d_out_flags, stream),
				"aclb200_decompress_tracks_inertialized");
		}
		// the same as skinning rows (aclb200_decompress_tracks_inertialized_skinning)
		void decompress_tracks_inertialized_skinning(const aclb200_inertialized_request* d_requests, uint32_t num_requests,
			const aclb200_options& options, const void* d_records, uint64_t num_records, const uint32_t* d_parent_indices, const float* d_inverse_bind,
			void* d_out, uint64_t record_stride_bytes = 0, const uint32_t* d_skeleton_offsets = nullptr, uint32_t* d_out_flags = nullptr,
			void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_inertialized_skinning(m_device->get(), m_clipset, d_requests, num_requests, &options, d_records,
				num_records, record_stride_bytes, d_parent_indices, d_skeleton_offsets, d_inverse_bind, d_out, d_out_flags, stream),
				"aclb200_decompress_tracks_inertialized_skinning");
		}
		// Each QVV48 pose of num_rows rows mirrored with d_table across the plane normal to `axis` (aclb200_mirror_poses); d_mirrored per
		// pose: 0 copies, 1 mirrors, other values leave the pose unwritten, NULL mirrors every pose. d_out may be d_poses.
		void mirror_poses(const void* d_poses, void* d_out, uint64_t num_poses, uint32_t num_rows, const aclb200_mirror_entry* d_table, uint32_t axis,
			const uint32_t* d_mirrored = nullptr, uint64_t pose_stride_bytes = 0, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_mirror_poses(m_device->get(), d_poses, d_out, num_poses, num_rows, pose_stride_bytes, d_mirrored, d_table, axis,
				d_out_flags, stream), "aclb200_mirror_poses");
		}
		// Decode and mirror in one launch (aclb200_decompress_tracks_mirrored): local rows without parents, object space rows of
		// `object_kind` with them; requests with mirrored == 0 as the plain decodes write them
		void decompress_tracks_mirrored(const aclb200_mirrored_request* d_requests, uint32_t num_requests, const aclb200_options& options,
			const aclb200_mirror_entry* d_mirror_table, uint32_t axis, void* d_out, const uint32_t* d_parent_indices = nullptr,
			const uint32_t* d_skeleton_offsets = nullptr, uint32_t object_kind = ACLB200_OBJECT_QVVF, uint32_t* d_out_flags = nullptr,
			void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_mirrored(m_device->get(), m_clipset, d_requests, num_requests, &options, d_mirror_table, axis,
				d_parent_indices, d_skeleton_offsets, object_kind, d_out, d_out_flags, stream), "aclb200_decompress_tracks_mirrored");
		}
		// the same as skinning rows (aclb200_decompress_tracks_mirrored_skinning)
		void decompress_tracks_mirrored_skinning(const aclb200_mirrored_request* d_requests, uint32_t num_requests, const aclb200_options& options,
			const aclb200_mirror_entry* d_mirror_table, uint32_t axis, const uint32_t* d_parent_indices, const float* d_inverse_bind, void* d_out,
			const uint32_t* d_skeleton_offsets = nullptr, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_decompress_tracks_mirrored_skinning(m_device->get(), m_clipset, d_requests, num_requests, &options, d_mirror_table,
				axis, d_parent_indices, d_skeleton_offsets, d_inverse_bind, d_out, d_out_flags, stream), "aclb200_decompress_tracks_mirrored_skinning");
		}
		// over num_poses QVV48 poses of one skeleton already on the device (aclb200_local_to_skinning); d_out may be d_local_poses
		void local_to_skinning(const void* d_local_poses, void* d_out, uint64_t num_poses, uint32_t num_tracks, const uint32_t* d_parent_indices,
			const float* d_inverse_bind, uint64_t pose_stride_bytes = 0, uint32_t* d_out_flags = nullptr, void* stream = nullptr)
		{
			m_device->check(aclb200_local_to_skinning(m_device->get(), d_local_poses, d_out, num_poses, num_tracks, pose_stride_bytes, d_parent_indices,
				d_inverse_bind, d_out_flags, stream), "aclb200_local_to_skinning");
		}
		// host buffers in, host buffers out, synchronous
		void decompress_tracks_host(const aclb200_request* requests, uint32_t num_requests, const aclb200_options& options, void* out, size_t out_bytes)
		{
			m_device->check(aclb200_decompress_tracks_host(m_device->get(), m_clipset, requests, num_requests, &options, out, out_bytes), "aclb200_decompress_tracks_host");
		}

	private:
		device_context* m_device;
		aclb200_clipset* m_clipset = nullptr;
		aclb200_clipset_info m_info = {};
	};

	// Drop-in for acl::database_context<database_settings> (decompression/database/database.h:85-170) over a database whose bulk data is
	// inline: initialize() streams every chunk in, as the reference's streamer-less initialize does (database.impl.h:91-212), and
	// stream_in / stream_out(tier, n) then move chunks of the inline bulk data in and out of HBM (aclb200_database_stream_in / _out).
	template<class database_settings_type = default_database_settings>
	class database_context
	{
	public:
		database_context() : m_device(&device_context::default_device()) {}
		explicit database_context(device_context& device) : m_device(&device) {}
		~database_context() { reset(); }
		database_context(const database_context&) = delete;
		database_context& operator=(const database_context&) = delete;

		// false for an invalid database or one whose bulk data is not inline (the reference asserts and returns false, :95-102)
		bool initialize(const compressed_database& database)
		{
			if (is_initialized())
				return false;
			aclb200_database* handle = nullptr;
			const aclb200_status status = aclb200_upload_database(m_device->get(), &database, database.get_size(), 0, &handle);
			if (status == ACLB200_ERR_INVALID_CLIP)
				return false;
			m_device->check(status, "aclb200_upload_database");
			m_device->check(aclb200_database_get_info(handle, &m_info), "aclb200_database_get_info");
			if (!m_info.is_bulk_data_inline)
			{
				aclb200_release_database(m_device->get(), handle);
				return false;
			}
			m_database = &database;
			m_handle = handle;
			for (uint32_t tier = ACLB200_TIER_MEDIUM; tier <= ACLB200_TIER_LOW; ++tier)
				if (m_info.num_chunks[tier - 1] != 0)
					m_device->check(aclb200_database_stream_in(m_device->get(), m_handle, tier, ~0u, nullptr, nullptr, nullptr), "aclb200_database_stream_in");
			return true;
		}
		void reset()
		{
			if (m_handle != nullptr)
				aclb200_release_database(m_device->get(), m_handle);
			m_handle = nullptr;
			m_database = nullptr;
		}
		bool is_initialized() const { return m_handle != nullptr; }
		const compressed_database* get_compressed_database() const { return m_database; }

		// database_context::contains, database.impl.h:369-405: the clip is bound to a database and its runtime clip header holds its hash
		bool contains(const compressed_tracks& tracks) const
		{
			if (!is_initialized())
				return false;
			const uint8_t* clip = reinterpret_cast<const uint8_t*>(&tracks);
			const uint8_t* db = reinterpret_cast<const uint8_t*>(m_database);
			if ((read32(clip + 28) & (1u << 8)) == 0)		// tracks_header::misc_packed bit 8, has_database
				return false;
			const uint32_t clip_header_offset = read32(clip + 32 + read32(clip + 32 + 32));	// transform_tracks_header::database_header_offset
			const uint32_t clip_metadata = 8 + read32(db + 8 + 28);
			for (uint32_t index = 0; index < m_info.num_clips; ++index)
				if (read32(db + clip_metadata + index * 8 + 4) == clip_header_offset && read32(db + clip_metadata + index * 8) == tracks.get_hash())
					return true;
			return false;
		}
		bool is_streamed_in(quality_tier tier) const
		{
			uint32_t loaded = 0;
			if (!is_initialized() || aclb200_database_get_loaded_chunks(m_handle, static_cast<uint32_t>(tier), &loaded) != ACLB200_OK)
				return false;
			return loaded == m_info.num_chunks[static_cast<uint32_t>(tier) - 1];
		}
		bool is_streaming(quality_tier) const { return false; }		// requests complete before stream_in / stream_out return
		database_stream_request_result stream_in(quality_tier tier, uint32_t num_chunks_to_stream = ~0u) { return stream(tier, num_chunks_to_stream, true); }
		database_stream_request_result stream_out(quality_tier tier, uint32_t num_chunks_to_stream = ~0u) { return stream(tier, num_chunks_to_stream, false); }

		const aclb200_database* handle() const { return m_handle; }

	private:
		static uint32_t read32(const uint8_t* p) { uint32_t v; std::memcpy(&v, p, 4); return v; }
		database_stream_request_result stream(quality_tier tier, uint32_t num_chunks, bool in)
		{
			if (!is_initialized())
				return database_stream_request_result::context_not_initialized;
			const uint32_t index = static_cast<uint32_t>(tier);
			if (index != ACLB200_TIER_MEDIUM && index != ACLB200_TIER_LOW)
				return database_stream_request_result::invalid_database_tier;
			if (m_info.num_chunks[index - 1] == 0)
				return database_stream_request_result::done;		// database.impl.h:485-486: nothing to stream
			uint32_t count = 0;
			const aclb200_status status = in ? aclb200_database_stream_in(m_device->get(), m_handle, index, num_chunks, nullptr, &count, nullptr)
				: aclb200_database_stream_out(m_device->get(), m_handle, index, num_chunks, &count, nullptr);
			m_device->check(status, in ? "aclb200_database_stream_in" : "aclb200_database_stream_out");
			return count != 0 ? database_stream_request_result::dispatched : database_stream_request_result::done;
		}

		device_context* m_device;
		const compressed_database* m_database = nullptr;
		aclb200_database* m_handle = nullptr;
		aclb200_database_info m_info = {};
	};

	// Where a batch writes its poses: device memory, request r at d_poses + r * pose_stride_bytes (0 = packed)
	struct device_pose_writer : track_writer
	{
		void* d_poses = nullptr;
		uint32_t output_layout = ACLB200_LAYOUT_QVV48;
		uint64_t pose_stride_bytes = 0;
		void* stream = nullptr;		// cudaStream_t
		// sub-tracks the batch does not write (track_writer::skip_all_* / skip_track_*): ACLB200_SKIP_* bits for every track, and an
		// optional device array of per track bits
		uint32_t skip_mask = 0;
		const uint8_t* d_skip_track_mask = nullptr;
	};

	// The batched form of decompression_context<settings>: bind N clips, seek N' (clip, time) requests, decode them in one launch.
	// The settings type plays the role it plays in the reference (decompress.h:76-88): it fixes the normalisation policy, wrapping,
	// per track rounding and sample time clamping at compile time.
	template<class settings_type = default_transform_decompression_settings>
	class batch_context
	{
		static_assert(std::is_base_of<decompression_settings, settings_type>::value, "settings_type must derive from decompression_settings");

	public:
		batch_context() : m_batch(device_context::default_device()) {}
		explicit batch_context(device_context& device) : m_batch(device) {}

		// initialize() for every clip of the batch; false (and the offending index) when one is not a valid compressed_tracks
		bool bind(const void* const* compressed_tracks_buffers, const uint32_t* sizes, uint32_t num_clips, uint32_t* out_failed_clip = nullptr)
		{
			m_num_requests = 0;
			return m_batch.upload(compressed_tracks_buffers, sizes, num_clips, true, out_failed_clip);
		}
		void reset() { m_batch.release(); m_num_requests = 0; }
		bool is_initialized() const { return m_batch.clipset() != nullptr; }
		uint32_t get_num_clips() const { return m_batch.info().num_clips; }
		uint32_t get_max_num_tracks() const { return m_batch.info().max_tracks; }
		void set_looping_policy(sample_looping_policy policy) { m_looping = policy; }
		sample_looping_policy get_looping_policy() const { return m_looping; }

		// seek() for a batch: d_requests is a DEVICE array of { clip index, sample_time }; evaluated on the GPU with the decode.
		// d_request_policies (optional): DEVICE [num_requests][2] bytes { rounding, looping } when the policies differ per request.
		void seek(const aclb200_request* d_requests, uint32_t num_requests, sample_rounding_policy rounding_policy, const uint8_t* d_request_policies = nullptr)
		{
			m_requests = d_requests;
			m_num_requests = num_requests;
			m_rounding = rounding_policy;
			m_request_policies = d_request_policies;
		}

		// decompress_tracks() for the batch, asynchronous on writer.stream
		template<class writer_type>
		void decompress_tracks(const writer_type& writer, const uint8_t* d_per_track_rounding = nullptr, const float* d_variable_defaults = nullptr)
		{
			if (!is_initialized() || m_num_requests == 0)
				return;
			aclb200_options options = make_options<settings_type>(writer, m_rounding, m_looping);
			// unlike the one pose shim, variable defaults live on the device here
			options.default_rotation_mode = static_cast<uint32_t>(writer_type::get_default_rotation_mode());
			options.default_translation_mode = static_cast<uint32_t>(writer_type::get_default_translation_mode());
			options.default_scale_mode = static_cast<uint32_t>(writer_type::get_default_scale_mode());
			options.d_variable_defaults = d_variable_defaults;
			options.d_per_track_rounding = d_per_track_rounding;
			options.d_request_policies = m_request_policies;
			options.output_layout = writer.output_layout;
			options.pose_stride_bytes = writer.pose_stride_bytes;
			options.skip_mask = writer.skip_mask | (writer_type::skip_all_rotations() ? uint32_t(ACLB200_SKIP_ROTATION) : 0u)
				| (writer_type::skip_all_translations() ? uint32_t(ACLB200_SKIP_TRANSLATION) : 0u) | (writer_type::skip_all_scales() ? uint32_t(ACLB200_SKIP_SCALE) : 0u);
			options.d_skip_track_mask = writer.d_skip_track_mask;
			m_batch.decompress_tracks(m_requests, m_num_requests, options, writer.d_poses, writer.stream);
		}

		batch_decompressor& decompressor() { return m_batch; }

	private:
		batch_decompressor m_batch;
		const aclb200_request* m_requests = nullptr;
		const uint8_t* m_request_policies = nullptr;
		uint32_t m_num_requests = 0;
		sample_looping_policy m_looping = sample_looping_policy::as_compressed;
		sample_rounding_policy m_rounding = sample_rounding_policy::none;
	};

	// Drop-in for acl::decompression_context<settings> (decompress.h:76-201): one clip bound, one pose per decompress_tracks().
	template<class decompression_settings_type = default_transform_decompression_settings>
	class decompression_context
	{
		static_assert(std::is_base_of<decompression_settings, decompression_settings_type>::value, "decompression_settings_type must derive from decompression_settings!");		// decompress.h:197

	public:
		using settings_type = decompression_settings_type;

		// decompress.h:90-95: default constructible; the GPU (device 0) is attached on first use
		decompression_context() : m_batch() {}
		explicit decompression_context(device_context& device) : m_batch(new batch_decompressor(device)) {}
		decompression_context(const decompression_context&) = delete;
		decompression_context& operator=(const decompression_context&) = delete;

		// initialize(const compressed_tracks&), decompress.impl.h:66-83 + initialize_v0 (decompression.transform.h:84-132):
		// false when the buffer is not a valid compressed_tracks, or when its version / track type / sub-track formats are not
		// among the ones the settings support
		bool initialize(const compressed_tracks& tracks)
		{
			reset();
			const uint32_t size = tracks.get_size();
			const uint32_t track_type = shim_impl::track_type_number(tracks.get_track_type());
			const uint32_t version = shim_impl::version_number(tracks.get_version());
			const uint32_t supported_version = shim_impl::version_number(settings_type::version_supported());
			if (!settings_type::skip_initialize_safety_checks())
			{
				if (supported_version != 0 && version != supported_version)
					return false;		// decompression_version_selector<version>::is_version_supported
				if (!shim_impl::supports_track_type<settings_type>(track_type))
					return false;
				if (track_type == ACLB200_TRACK_QVVF && size >= 32)
				{
					// tracks_header::misc_packed (core/impl/compressed_headers.h:95-124): bit 2 scale format, bit 3 translation format, bits 4-7 rotation format
					const uint32_t misc = shim_impl::read_u32(&tracks, 28);
					if (!shim_impl::supports_rotation_format<settings_type>((misc >> 4) & 15u) || !shim_impl::supports_translation_format<settings_type>((misc >> 3) & 1u)
						|| ((misc & 1u) != 0 && !shim_impl::supports_scale_format<settings_type>((misc >> 2) & 1u)))
						return false;
				}
			}
			const void* blobs[1] = { &tracks };
			const uint32_t sizes[1] = { size };
			if (!batch().upload(blobs, sizes, 1, /*check_hash*/ false))		// the reference's initialize() runs is_valid(false) as well
				return false;
			m_bound = &tracks;
			m_hash = tracks.get_hash();
			m_looping = sample_looping_policy::as_compressed;
			m_has_seeked = false;
			const aclb200_clipset_info& info = batch().info();
			m_components = info.track_type == ACLB200_TRACK_QVVF ? 12u : (info.track_type <= 3 ? info.track_type + 1 : 4u);
			m_pose.assign(size_t(info.max_tracks) * m_components, 0.0F);
			return true;
		}
		// initialize(tracks, database), decompress.impl.h:85-110: false when the database does not contain the clip; the clip then decodes
		// from the tiers of `database` streamed in, at the time of each decompress call
		template<class database_settings_type>
		bool initialize(const compressed_tracks& tracks, const database_context<database_settings_type>& database)
		{
			if (!database.is_initialized() || !database.contains(tracks) || !initialize(tracks))
				return false;
			if (!batch().bind_database(database.handle()))
			{
				reset();
				return false;
			}
			return true;
		}
		// a raw buffer holding a compressed_tracks instance
		bool initialize(const void* compressed_tracks_buffer, uint32_t /*size*/ = 0)
		{
			return compressed_tracks_buffer != nullptr && initialize(*static_cast<const compressed_tracks*>(compressed_tracks_buffer));
		}

		// relocated(const compressed_tracks&), decompress.impl.h:119-137 + relocated_v0 (decompression.transform.h:134-157): the clip
		// moved in host memory. Only the SAME clip is accepted (same hash); the device copy is unaffected.
		bool relocated(const compressed_tracks& tracks)
		{
			if (!is_initialized())
				return false;
			if (tracks.get_hash() != m_hash || tracks.get_size() != batch_info_size())
				return false;		// Hash is different, this instance did not relocate, it is different
			m_bound = &tracks;
			return true;
		}
		void reset()		// decompress.h:120-124
		{
			if (m_batch)
				m_batch->release();
			m_bound = nullptr;
			m_has_seeked = false;
		}
		const compressed_tracks* get_compressed_tracks() const { return m_bound; }
		bool is_initialized() const { return m_bound != nullptr; }
		// the device side of the bound clip (a clip set of one), for the callers of the decode that run on the device as well
		// (acl_b200/track_error.h)
		batch_decompressor& device_batch() { return batch(); }
		// is_bound_to_v0, decompression.transform.h:159-176: same address and same hash
		bool is_bound_to(const compressed_tracks& tracks) const { return m_bound == &tracks && m_hash == tracks.get_hash(); }
		void set_looping_policy(sample_looping_policy policy)
		{
			if (is_initialized())
				m_looping = policy;
		}
		sample_looping_policy get_looping_policy() const { return m_looping; }

		// seek(), decompress.impl.h:207-222: remembered here, evaluated on the GPU together with the decode
		void seek(float sample_time, sample_rounding_policy rounding_policy)
		{
			if (!is_initialized())
				return;		// ACL_ASSERT(m_context.is_initialized()) then nothing
			if (rounding_policy == sample_rounding_policy::per_track && !settings_type::is_per_track_rounding_supported())
				return;		// ACL_ASSERT in the reference (decompress.impl.h:211): the seek does not happen
			m_sample_time = sample_time;
			m_rounding = rounding_policy;
			m_has_seeked = true;
		}

		template<class track_writer_type>
		void decompress_tracks(track_writer_type& writer)
		{
			static_assert(std::is_base_of<track_writer, track_writer_type>::value, "track_writer_type must derive from track_writer");		// decompress.impl.h:228
			if (!is_initialized() || !m_has_seeked)
				return;		// the reference asserts; like it, nothing is written
			const uint32_t num_tracks = batch().info().max_tracks;
			if (num_tracks == 0)
				return;		// empty track list: nothing to do (decompression.transform.h:1535-1537)
			aclb200_options options = make_options<settings_type>(writer, m_rounding, m_looping);
			if (m_components != 12)
			{
				decode_pose(writer, options);
				for (uint32_t track = 0; track < num_tracks; ++track)
					replay_scalar(writer, track, m_pose.data() + size_t(track) * m_components);
				return;
			}
			prime_skipped(options, num_tracks);
			decode_pose(writer, options);
			for (uint32_t track = 0; track < num_tracks; ++track)
				replay(writer, options, track, m_pose.data() + size_t(track) * 12);
		}

		// decompress_track(track_index, writer): the batched decompress_track_v0 kernel (decompression.transform.h:1753-2050,
		// decompression.scalar.h:483-705) on ONE request: one bone / track crosses PCIe, not the pose
		template<class track_writer_type>
		void decompress_track(uint32_t track_index, track_writer_type& writer)
		{
			static_assert(std::is_base_of<track_writer, track_writer_type>::value, "track_writer_type must derive from track_writer");
			if (!is_initialized() || !m_has_seeked || track_index >= batch().info().max_tracks)
				return;
			device_context& device = batch().device();
			aclb200_options options = make_options<settings_type>(writer, m_rounding, m_looping);
			uint8_t track_policy = 0;
			if (m_rounding == sample_rounding_policy::per_track)
				track_policy = static_cast<uint8_t>(writer.get_rounding_policy(m_rounding, track_index));
			const bool transform = m_components == 12;
			const size_t value_bytes = (transform ? 12 : m_components) * sizeof(float);
			// device scratch: request | track index | this track's policy replicated for every track index | value
			const uint32_t num_tracks = batch().info().max_tracks;
			const size_t policy_offset = 16, value_offset = (policy_offset + num_tracks + 15) & ~size_t(15);
			uint8_t* scratch = static_cast<uint8_t*>(m_track_scratch.get(device, value_offset + 64));
			std::vector<uint8_t> staging(value_offset, 0);
			const aclb200_request request = { 0u, m_sample_time };
			std::memcpy(staging.data(), &request, sizeof(request));
			std::memcpy(staging.data() + 8, &track_index, 4);
			std::memset(staging.data() + policy_offset, track_policy, num_tracks);
			float bone[16];
			if (transform)
			{
				prime_skipped_bone(options, bone);
				device.check(aclb200_copy_to_device(device.get(), scratch + value_offset, bone, value_bytes), "aclb200_copy_to_device");
			}
			if (m_rounding == sample_rounding_policy::per_track)
				options.d_per_track_rounding = scratch + policy_offset;
			device.check(aclb200_copy_to_device(device.get(), scratch, staging.data(), staging.size()), "aclb200_copy_to_device");
			batch().decompress_track(reinterpret_cast<const aclb200_request*>(scratch), reinterpret_cast<const uint32_t*>(scratch + 8), 1, options, scratch + value_offset);
			device.check(aclb200_copy_to_host(device.get(), bone, scratch + value_offset, value_bytes), "aclb200_copy_to_host");
			if (transform)
				replay(writer, options, track_index, bone);
			else
				replay_scalar(writer, track_index, bone);
		}

	private:
		batch_decompressor& batch()
		{
			if (!m_batch)
				m_batch.reset(new batch_decompressor(device_context::default_device()));
			return *m_batch;
		}
		const batch_decompressor& batch() const { return *m_batch; }
		uint32_t batch_info_size() const
		{
			aclb200_clip_info info = {};
			return aclb200_clipset_get_clip_info(m_batch->clipset(), 0, &info) == ACLB200_OK ? info.size : 0u;
		}

		// one pose through the host buffer entry point; per_track rounding asks the writer for every track's policy first
		template<class track_writer_type>
		void decode_pose(track_writer_type& writer, aclb200_options& options)
		{
			device_context& device = batch().device();
			if (m_rounding == sample_rounding_policy::per_track)
			{
				const uint32_t num_tracks = batch().info().max_tracks;
				std::vector<uint8_t> policies(num_tracks);
				for (uint32_t track = 0; track < num_tracks; ++track)
					policies[track] = static_cast<uint8_t>(writer.get_rounding_policy(m_rounding, track));		// core/track_writer.h:90
				void* d_policies = m_policy_scratch.get(device, num_tracks);
				device.check(aclb200_copy_to_device(device.get(), d_policies, policies.data(), num_tracks), "aclb200_copy_to_device");
				options.d_per_track_rounding = static_cast<const uint8_t*>(d_policies);
			}
			const aclb200_request request = { 0u, m_sample_time };
			batch().decompress_tracks_host(&request, 1, options, m_pose.data(), m_pose.size() * sizeof(float));
		}

		// `skipped` default sub-tracks are left untouched by the device: mark them so the replay can tell them from written ones
		static constexpr uint32_t k_marker = 0x7FC0ACB2u;		// a NaN payload no decode produces
		static bool any_skipped(const aclb200_options& options)
		{
			return options.default_rotation_mode == ACLB200_DEFAULT_SKIPPED || options.default_translation_mode == ACLB200_DEFAULT_SKIPPED
				|| options.default_scale_mode == ACLB200_DEFAULT_SKIPPED;
		}
		void prime_skipped(const aclb200_options& options, uint32_t num_tracks)
		{
			if (!any_skipped(options))
				return;
			const uint32_t marker = k_marker;
			for (uint32_t i = 0; i < num_tracks * 12; ++i)
				std::memcpy(&m_pose[i], &marker, sizeof(marker));
		}
		static void prime_skipped_bone(const aclb200_options&, float bone[12])
		{
			const uint32_t marker = k_marker;
			for (uint32_t i = 0; i < 12; ++i)
				std::memcpy(&bone[i], &marker, sizeof(marker));
		}
		static bool is_marker(const float* v)
		{
			uint32_t bits;
			std::memcpy(&bits, v, sizeof(bits));
			return bits == k_marker;
		}

		template<class track_writer_type>
		static void replay(track_writer_type& writer, const aclb200_options& options, uint32_t track, const float* bone)
		{
			if (!track_writer_type::skip_all_rotations() && !writer.skip_track_rotation(track))
			{
				if (!(options.default_rotation_mode == ACLB200_DEFAULT_SKIPPED && is_marker(bone)))
					writer.write_rotation(track, shim_impl::make_rotation(bone));
				else if (track_writer_type::get_default_rotation_mode() == default_sub_track_mode::variable)
					writer.write_rotation(track, writer.get_variable_default_rotation(track));
			}
			if (!track_writer_type::skip_all_translations() && !writer.skip_track_translation(track))
			{
				if (!(options.default_translation_mode == ACLB200_DEFAULT_SKIPPED && is_marker(bone + 4)))
					writer.write_translation(track, shim_impl::make_vector(bone + 4));
				else if (track_writer_type::get_default_translation_mode() == default_sub_track_mode::variable)
					writer.write_translation(track, writer.get_variable_default_translation(track));
			}
			if (!track_writer_type::skip_all_scales() && !writer.skip_track_scale(track))
			{
				if (!(options.default_scale_mode == ACLB200_DEFAULT_SKIPPED && is_marker(bone + 8)))
					writer.write_scale(track, shim_impl::make_vector(bone + 8));
				else if (track_writer_type::get_default_scale_mode() == default_sub_track_mode::variable)
					writer.write_scale(track, writer.get_variable_default_scale(track));
			}
		}

		// scalar clips: write_float1 .. write_float4 / write_vector4 (decompression.scalar.h:289-470)
		template<class track_writer_type>
		void replay_scalar(track_writer_type& writer, uint32_t track, const float* value) const
		{
			float padded[4] = { 0.0F, 0.0F, 0.0F, 0.0F };
			std::memcpy(padded, value, m_components * sizeof(float));
			switch (batch().info().track_type)
			{
			case ACLB200_TRACK_FLOAT1F:
				if (!writer.skip_track_float1(track))
					writer.write_float1(track, shim_impl::make_scalar(padded));
				break;
			case ACLB200_TRACK_FLOAT2F:
				if (!writer.skip_track_float2(track))
					writer.write_float2(track, shim_impl::make_vector(padded));
				break;
			case ACLB200_TRACK_FLOAT3F:
				if (!writer.skip_track_float3(track))
					writer.write_float3(track, shim_impl::make_vector(padded));
				break;
			case ACLB200_TRACK_FLOAT4F:
				if (!writer.skip_track_float4(track))
					writer.write_float4(track, shim_impl::make_vector(padded));
				break;
			default:
				if (!writer.skip_track_vector4(track))
					writer.write_vector4(track, shim_impl::make_vector(padded));
				break;
			}
		}

		std::unique_ptr<batch_decompressor> m_batch;
		const compressed_tracks* m_bound = nullptr;
		uint32_t m_hash = 0;
		uint32_t m_components = 12;
		sample_looping_policy m_looping = sample_looping_policy::as_compressed;
		sample_rounding_policy m_rounding = sample_rounding_policy::none;
		float m_sample_time = 0.0F;
		bool m_has_seeked = false;
		std::vector<float> m_pose;
		shim_impl::device_buffer m_policy_scratch, m_track_scratch;
	};
}
