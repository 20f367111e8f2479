// acl_b200/csrc/database.cpp -- streaming databases on the device: aclb200_upload_database validates a compressed_database blob,
// stream_in / stream_out move chunks of its medium and low importance tiers in and out of HBM, and aclb200_clipset_bind_database binds a
// clip set to it. The seek of the database kernels (device_common.cuh seek_transform<true>) reads what is kept here:
//
//   d_tiers   u64[num_segments][2]   database_runtime_segment_header::tier_metadata (core/impl/compressed_headers.h:404-422) of every
//                                    database segment, in runtime header order: (samples_offset << 32) | sample_indices, 0 when the
//                                    chunk holding the segment is not streamed in
//   d_bulk[t] tier buffer            the tier's bulk data, stored as the clip streams are (layout.h): byte-swapped 32-bit words over the
//                                    whole buffer from offset 0, plus k_stream_tail bytes of slack for the two-word reads
//
// Chunk selection, allocation and release follow database_context::stream_in / stream_out (decompression/database/impl/database.impl.h:
// 443-637) with a streamer that copies synchronously, like the reference's debug_database_streamer.
#include "context.h"

#include <algorithm>
#include <cstring>
#include <new>

namespace aclb200
{
	namespace
	{
		inline uint32_t rd_u32(const uint8_t* p) { uint32_t v; std::memcpy(&v, p, 4); return v; }
		inline uint16_t rd_u16(const uint8_t* p) { uint16_t v; std::memcpy(&v, p, 2); return v; }

		constexpr uint32_t k_database_tag = 0xac11db01u;			// buffer_tag32::compressed_database, core/buffer_tag.h:53
		constexpr uint32_t k_header_offset = 8;						// raw_buffer_header { size, hash }
		constexpr uint32_t k_header_size = 56;						// database_header, compressed_headers.h:540-573
		constexpr uint32_t k_chunk_header_size = 12;				// database_chunk_header { index, size, num_segments }
		constexpr uint32_t k_chunk_segment_header_size = 20;		// database_chunk_segment_header
		constexpr uint32_t k_runtime_clip_header_size = 8;			// database_runtime_clip_header
		constexpr uint32_t k_runtime_segment_header_size = 16;		// database_runtime_segment_header

		// core/hash.h:44-84 (FNV-1a 32)
		uint32_t hash32(const uint8_t* data, size_t size)
		{
			uint32_t acc = 2166136261u;
			for (size_t i = 0; i < size; ++i)
				acc = (acc ^ data[i]) * 16777619u;
			return acc;
		}

		// acl::bitset: bit i lives in word i / 32 at (31 - i % 32)
		void bit_set(std::vector<uint32_t>& bits, uint32_t i, bool value)
		{
			const uint32_t mask = 1u << (31 - i % 32);
			bits[i / 32] = value ? (bits[i / 32] | mask) : (bits[i / 32] & ~mask);
		}
		uint32_t bit_count(const std::vector<uint32_t>& bits)
		{
			uint32_t count = 0;
			for (uint32_t word : bits)
				count += uint32_t(__builtin_popcount(word));
			return count;
		}

		// Flat database segment index of a runtime segment header offset, or 0xFFFFFFFF when the offset names no segment header
		uint32_t segment_at(const aclb200_database& db, const std::vector<uint32_t>& by_offset, uint32_t offset)
		{
			auto it = std::upper_bound(by_offset.begin(), by_offset.end(), offset,
				[&](uint32_t value, uint32_t clip) { return value < db.clip_header_offset[clip]; });
			if (it == by_offset.begin())
				return 0xFFFFFFFFu;
			const uint32_t clip = *(it - 1);
			const uint64_t relative = uint64_t(offset) - db.clip_header_offset[clip];
			if (relative < k_runtime_clip_header_size || (relative - k_runtime_clip_header_size) % k_runtime_segment_header_size != 0)
				return 0xFFFFFFFFu;
			const uint32_t segment = uint32_t((relative - k_runtime_clip_header_size) / k_runtime_segment_header_size);
			return segment < db.clip_num_segments[clip] ? db.clip_first_segment[clip] + segment : 0xFFFFFFFFu;
		}

		struct published
		{
			uint32_t segment;
			uint64_t metadata;
		};

		// The segments of chunk `chunk` of tier `t` and their tier metadata, read from the tier's bulk data as database.impl.h:160-210
		// does; every offset is checked against the tier so that no key frame read can leave the tier buffer. Empty string: valid.
		std::string read_chunk(const aclb200_database& db, const std::vector<uint32_t>& by_offset, uint32_t t, uint32_t chunk,
			const uint8_t* bulk, std::vector<published>& out)
		{
			const uint32_t description = k_header_offset + (t == 0 ? k_header_size : ((k_header_size + db.info.num_chunks[0] * 8 + 3) & ~3u)) + chunk * 8;
			const uint32_t chunk_size = rd_u32(db.blob.data() + description);
			const uint32_t chunk_offset = rd_u32(db.blob.data() + description + 4);
			const uint64_t bulk_size = db.info.bulk_data_size[t];
			const uint8_t* p = bulk + chunk_offset;
			if (rd_u32(p) != chunk)
				return "chunk header index does not match its description";
			const uint32_t num_segments = rd_u32(p + 8);
			if (k_chunk_header_size + uint64_t(num_segments) * k_chunk_segment_header_size > chunk_size)
				return "chunk segment headers exceed the chunk";
			for (uint32_t i = 0; i < num_segments; ++i)
			{
				const uint8_t* s = p + k_chunk_header_size + i * k_chunk_segment_header_size;
				const uint32_t sample_indices = rd_u32(s + 4);
				const uint32_t samples_offset = rd_u32(s + 8);
				const uint32_t segment = segment_at(db, by_offset, rd_u32(s + 16));
				if (segment == 0xFFFFFFFFu)
					return "chunk segment names no runtime segment header";
				if (samples_offset > bulk_size)
					return "chunk segment samples out of bounds";
				const uint32_t pose_bits = db.segment_pose_bits[segment];
				if (pose_bits != 0 && samples_offset + (uint64_t(pose_bits) * uint32_t(__builtin_popcount(sample_indices)) + 7) / 8 > bulk_size)
					return "chunk segment samples out of bounds";
				out.push_back({ segment, (uint64_t(samples_offset) << 32) | sample_indices });
			}
			return std::string();
		}

		std::vector<uint32_t> clips_by_offset(const aclb200_database& db)
		{
			std::vector<uint32_t> order(db.info.num_clips);
			for (uint32_t i = 0; i < db.info.num_clips; ++i)
				order[i] = i;
			std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return db.clip_header_offset[a] < db.clip_header_offset[b]; });
			return order;
		}

		// Copies the tier t entries of the given segments to d_tiers: one strided copy per run of consecutive segments, so the
		// other tier's entries are never written (a stream_in of one tier may run on another stream than one of the other tier)
		cudaError_t publish(aclb200_database& db, uint32_t t, std::vector<uint32_t> segments, cudaStream_t stream)
		{
			std::sort(segments.begin(), segments.end());
			segments.erase(std::unique(segments.begin(), segments.end()), segments.end());
			cudaError_t error = cudaSuccess;
			for (size_t i = 0; i < segments.size() && error == cudaSuccess; )
			{
				size_t j = i + 1;
				while (j < segments.size() && segments[j] == segments[j - 1] + 1)
					++j;
				const size_t first = segments[i];
				error = cudaMemcpy2DAsync(db.d_tiers + 2 * first + t, 16, db.host_tiers.data() + 2 * first + t, 16, 8, j - i, cudaMemcpyHostToDevice, stream);
				i = j;
			}
			return error;
		}

		std::string validate(const uint8_t* blob, uint32_t size, bool check_hash, aclb200_database& db)
		{
			// compressed_database::is_valid, core/impl/compressed_database.impl.h:142-162
			if (size < k_header_offset + k_header_size)
				return "buffer too small";
			const uint32_t stored_size = rd_u32(blob);
			if (stored_size > size || stored_size < k_header_offset + k_header_size)
				return "stored size does not fit the buffer";
			const uint8_t* h = blob + k_header_offset;
			if (rd_u32(h + 0) != k_database_tag)
				return "invalid tag";
			const uint32_t version = rd_u16(h + 4);
			if (version < k_version_first || version > k_version_latest)
				return "invalid database version";
			if (check_hash && hash32(blob + 8, stored_size - 8) != rd_u32(blob + 4))
				return "invalid hash";

			aclb200_database_info& info = db.info;
			info.is_bulk_data_inline = rd_u16(h + 6) & 1u;
			info.num_chunks[0] = rd_u32(h + 8);
			info.num_chunks[1] = rd_u32(h + 12);
			info.max_chunk_size = rd_u32(h + 16);
			info.num_clips = rd_u32(h + 20);
			info.num_segments = rd_u32(h + 24);
			const uint32_t clip_metadata_offset = rd_u32(h + 28);
			info.bulk_data_size[0] = rd_u32(h + 32);
			info.bulk_data_size[1] = rd_u32(h + 36);
			info.hash = rd_u32(blob + 4);
			info.size = stored_size;
			auto in_blob = [&](uint64_t offset, uint64_t bytes) { return offset + bytes <= stored_size; };

			// chunk descriptions (database_header::get_chunk_descriptions_medium / _low, compressed_headers.h:590-596)
			const uint64_t descriptions[2] = { k_header_offset + k_header_size, k_header_offset + ((k_header_size + uint64_t(info.num_chunks[0]) * 8 + 3) & ~3ull) };
			for (uint32_t t = 0; t < 2; ++t)
			{
				if (!in_blob(descriptions[t], uint64_t(info.num_chunks[t]) * 8))
					return "chunk descriptions out of bounds";
				for (uint32_t chunk = 0; chunk < info.num_chunks[t]; ++chunk)
				{
					const uint32_t chunk_size = rd_u32(blob + descriptions[t] + chunk * 8);
					const uint32_t chunk_offset = rd_u32(blob + descriptions[t] + chunk * 8 + 4);
					if (chunk_size < k_chunk_header_size || chunk_size > info.max_chunk_size || uint64_t(chunk_offset) + chunk_size > info.bulk_data_size[t])
						return "chunk description out of bounds";
				}
				// stream_in / stream_out copy (n - 1) * max_chunk_size + the last chunk's size from the first chunk's offset
				if (info.num_chunks[t] != 0)
				{
					const uint64_t first = rd_u32(blob + descriptions[t] + 4);
					for (uint32_t chunk = 0; chunk < info.num_chunks[t]; ++chunk)
						if (first + uint64_t(chunk) * info.max_chunk_size + rd_u32(blob + descriptions[t] + chunk * 8) > info.bulk_data_size[t])
							return "chunk range out of bounds";
				}
				if (info.is_bulk_data_inline && info.bulk_data_size[t] != 0)
				{
					const uint32_t bulk_offset = rd_u32(h + 40 + 4 * t);
					if (bulk_offset == 0xFFFFFFFFu || !in_blob(uint64_t(k_header_offset) + bulk_offset, info.bulk_data_size[t]))
						return "inline bulk data out of bounds";
				}
			}

			// clip metadata and the runtime header layout they imply: [clip header, segment headers...] per clip
			if (!in_blob(uint64_t(k_header_offset) + clip_metadata_offset, uint64_t(info.num_clips) * 8))
				return "clip metadata out of bounds";
			const uint64_t runtime_size = uint64_t(info.num_clips) * k_runtime_clip_header_size + uint64_t(info.num_segments) * k_runtime_segment_header_size;
			db.clip_hash.resize(info.num_clips);
			db.clip_header_offset.resize(info.num_clips);
			db.clip_first_segment.resize(info.num_clips);
			db.clip_num_segments.resize(info.num_clips);
			for (uint32_t clip = 0; clip < info.num_clips; ++clip)
			{
				db.clip_hash[clip] = rd_u32(blob + k_header_offset + clip_metadata_offset + clip * 8);
				db.clip_header_offset[clip] = rd_u32(blob + k_header_offset + clip_metadata_offset + clip * 8 + 4);
			}
			const std::vector<uint32_t> order = clips_by_offset(db);
			uint64_t expected = 0;
			// build_database lists every segment of the database in the chunk headers of each tier that has chunks: a segment count past
			// what those headers can hold is a corrupt header (and would size the tier tables from garbage)
			uint64_t segment_capacity = 65536;
			for (uint32_t t = 0; t < 2; ++t)
			{
				uint64_t capacity = 0;
				for (uint32_t chunk = 0; chunk < info.num_chunks[t]; ++chunk)
					capacity += (rd_u32(blob + descriptions[t] + chunk * 8) - k_chunk_header_size) / k_chunk_segment_header_size;
				segment_capacity = capacity > segment_capacity ? capacity : segment_capacity;
			}
			if (info.num_segments > segment_capacity)
				return "more segments than the chunk headers can list";
			uint32_t segment = 0;
			for (uint32_t rank = 0; rank < info.num_clips; ++rank)
			{
				const uint32_t clip = order[rank];
				const uint64_t next = rank + 1 < info.num_clips ? db.clip_header_offset[order[rank + 1]] : runtime_size;
				if (db.clip_header_offset[clip] != expected || next < expected + k_runtime_clip_header_size
					|| (next - expected - k_runtime_clip_header_size) % k_runtime_segment_header_size != 0)
					return "clip metadata offsets do not tile the runtime headers";
				db.clip_first_segment[clip] = segment;
				db.clip_num_segments[clip] = uint32_t((next - expected - k_runtime_clip_header_size) / k_runtime_segment_header_size);
				segment += db.clip_num_segments[clip];
				expected = next;
			}
			if (segment != info.num_segments)
				return "segment count does not match the runtime headers";
			db.segment_pose_bits.assign(info.num_segments, 0u);

			// inline bulk data: every chunk header is checked now
			if (info.is_bulk_data_inline)
			{
				db.blob.assign(blob, blob + stored_size);
				for (uint32_t t = 0; t < 2; ++t)
					for (uint32_t chunk = 0; chunk < info.num_chunks[t]; ++chunk)
					{
						std::vector<published> entries;
						const std::string error = read_chunk(db, order, t, chunk, blob + k_header_offset + rd_u32(h + 40 + 4 * t), entries);
						if (!error.empty())
							return error;
					}
			}
			return std::string();
		}

		aclb200_status check_tier(aclb200_context* context, const aclb200_database* database, uint32_t tier, const char* what)
		{
			if (context == nullptr || database == nullptr)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": null context / database");
			if (tier != ACLB200_TIER_MEDIUM && tier != ACLB200_TIER_LOW)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": the tier must be ACLB200_TIER_MEDIUM or ACLB200_TIER_LOW");
			if (database->info.num_chunks[tier - 1] == 0)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": the tier has no chunks");
			if (database->device != context->device)
				return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, std::string(what) + ": the database lives on another device");
			return ACLB200_OK;
		}
	}

	bool database_streamed_in(const aclb200_clipset* clipset)
	{
		if (clipset == nullptr || clipset->database == nullptr)
			return false;
		return bit_count(clipset->database->loaded[0]) + bit_count(clipset->database->loaded[1]) != 0;
	}
}

using namespace aclb200;

extern "C"
{
	aclb200_status aclb200_upload_database(aclb200_context* context, const void* blob, uint32_t size, uint32_t check_hash, aclb200_database** out_database)
	{
		if (context == nullptr || blob == nullptr || out_database == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "upload_database: null argument");
		*out_database = nullptr;
		aclb200_database* db = new (std::nothrow) aclb200_database();
		if (db == nullptr)
			return set_error(context, ACLB200_ERR_OUT_OF_MEMORY, "upload_database: out of host memory");
		try
		{
			const std::string error = validate(static_cast<const uint8_t*>(blob), size, check_hash != 0, *db);
			if (!error.empty())
			{
				delete db;
				return set_error(context, ACLB200_ERR_INVALID_CLIP, "upload_database: " + error);
			}
			if (db->blob.empty())
				db->blob.assign(static_cast<const uint8_t*>(blob), static_cast<const uint8_t*>(blob) + db->info.size);
			db->host_tiers.assign(size_t(db->info.num_segments) * 2, 0);
			for (uint32_t t = 0; t < 2; ++t)
			{
				db->loaded[t].assign((db->info.num_chunks[t] + 31) / 32, 0u);
				db->chunk_segments[t].resize(db->info.num_chunks[t]);
			}
		}
		catch (const std::exception&)
		{
			delete db;
			return set_error(context, ACLB200_ERR_OUT_OF_MEMORY, "upload_database: out of host memory");
		}
		db->device = context->device;
		const size_t table_bytes = size_t(db->info.num_segments) * 16 + 16;
		cudaError_t error = cudaSetDevice(context->device);
		if (error == cudaSuccess) error = cudaMalloc(reinterpret_cast<void**>(&db->d_tiers), table_bytes);
		if (error == cudaSuccess) error = cudaMemset(db->d_tiers, 0, table_bytes);
		if (error != cudaSuccess)
		{
			cudaFree(db->d_tiers);
			delete db;
			return check_cuda(context, error, "upload_database");
		}
		*out_database = db;
		return ACLB200_OK;
	}

	void aclb200_release_database(aclb200_context* context, aclb200_database* database)
	{
		(void)context;
		if (database == nullptr)
			return;
		cudaSetDevice(database->device);
		cudaDeviceSynchronize();
		cudaFree(database->d_tiers);
		cudaFree(database->d_bulk[0]);
		cudaFree(database->d_bulk[1]);
		delete database;
	}

	aclb200_status aclb200_database_get_info(const aclb200_database* database, aclb200_database_info* out_info)
	{
		if (database == nullptr || out_info == nullptr)
			return ACLB200_ERR_INVALID_ARGUMENT;
		*out_info = database->info;
		return ACLB200_OK;
	}

	aclb200_status aclb200_database_get_loaded_chunks(const aclb200_database* database, uint32_t tier, uint32_t* out_loaded_chunks)
	{
		if (database == nullptr || out_loaded_chunks == nullptr || (tier != ACLB200_TIER_MEDIUM && tier != ACLB200_TIER_LOW))
			return ACLB200_ERR_INVALID_ARGUMENT;
		*out_loaded_chunks = bit_count(database->loaded[tier - 1]);
		return ACLB200_OK;
	}

	aclb200_status aclb200_database_stream_in(aclb200_context* context, aclb200_database* db, uint32_t tier, uint32_t num_chunks,
		const void* host_bulk_data, uint32_t* out_num_chunks, void* stream)
	{
		aclb200_status status = check_tier(context, db, tier, "database_stream_in");
		if (status != ACLB200_OK)
			return status;
		if (out_num_chunks != nullptr)
			*out_num_chunks = 0;
		const uint32_t t = tier - 1;
		const uint8_t* header = db->blob.data() + k_header_offset;
		const uint8_t* bulk = static_cast<const uint8_t*>(host_bulk_data);
		if (bulk == nullptr && db->info.is_bulk_data_inline)
			bulk = header + rd_u32(header + 40 + 4 * t);
		if (bulk == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "database_stream_in: the bulk data is not inline: pass the tier's bulk data");

		// the chunk range of database.impl.h:462-496: from the first chunk after the loaded ones, at most num_chunks
		const uint32_t tier_chunks = db->info.num_chunks[t];
		num_chunks = std::min(num_chunks, tier_chunks);
		uint32_t first_chunk = ~0u;
		for (size_t entry = 0; entry < db->loaded[t].size(); ++entry)
		{
			const uint32_t word = db->loaded[t][entry];
			const uint32_t pending = word == 0 ? 32u : uint32_t(__builtin_ctz(word));
			if (pending != 0)
			{
				first_chunk = uint32_t(entry) * 32 + (32 - pending);
				break;
			}
		}
		if (first_chunk == ~0u)
			return ACLB200_OK;
		const uint64_t last64 = uint64_t(first_chunk) + uint64_t(num_chunks) - 1;
		const uint32_t last_chunk = last64 >= uint64_t(tier_chunks) ? tier_chunks - 1 : uint32_t(last64);
		const uint32_t count = last_chunk - first_chunk + 1;
		if (count == 0 || last_chunk < first_chunk)
			return ACLB200_OK;

		try
		{
			const std::vector<uint32_t> order = clips_by_offset(*db);
			std::vector<published> entries;
			std::vector<size_t> chunk_end;
			for (uint32_t chunk = first_chunk; chunk <= last_chunk; ++chunk)
			{
				const std::string error = read_chunk(*db, order, t, chunk, bulk, entries);
				if (!error.empty())
					return set_error(context, ACLB200_ERR_INVALID_CLIP, "database_stream_in: chunk " + std::to_string(chunk) + ": " + error);
				chunk_end.push_back(entries.size());
			}

			// the bytes of the range, byte-swapped per 32-bit word: boundary words come whole from the caller's copy of the tier, so a
			// chunk streamed in later never needs a neighbour's bytes swapped again
			const uint32_t descriptions = k_header_offset + (t == 0 ? k_header_size : ((k_header_size + db->info.num_chunks[0] * 8 + 3) & ~3u));
			const uint64_t start = rd_u32(db->blob.data() + descriptions + first_chunk * 8 + 4);
			const uint64_t end = start + uint64_t(count - 1) * db->info.max_chunk_size + rd_u32(db->blob.data() + descriptions + last_chunk * 8);
			const uint64_t bulk_size = db->info.bulk_data_size[t];
			const uint64_t first_word = start / 4, end_word = (end + 3) / 4;
			std::vector<uint8_t> staging(size_t(end_word - first_word) * 4, 0);
			for (uint64_t i = first_word * 4; i < end_word * 4 && i < bulk_size; ++i)
				staging[size_t(i - first_word * 4 + (3 - 2 * (i & 3)))] = bulk[i];

			cudaStream_t cuda_stream = static_cast<cudaStream_t>(stream);
			cudaError_t error = cudaSetDevice(context->device);
			if (error == cudaSuccess && db->d_bulk[t] == nullptr)
			{
				// the words of chunks not streamed in yet are never read; the tail is zeroed like the clip streams' (layout.h k_stream_tail)
				const size_t padded = size_t((bulk_size + 3) & ~3ull);
				error = cudaMallocAsync(reinterpret_cast<void**>(&db->d_bulk[t]), padded + k_stream_tail, cuda_stream);
				if (error == cudaSuccess)
					error = cudaMemsetAsync(db->d_bulk[t] + padded, 0, k_stream_tail, cuda_stream);
			}
			if (error == cudaSuccess)
				error = cudaMemcpyAsync(db->d_bulk[t] + first_word * 4, staging.data(), staging.size(), cudaMemcpyHostToDevice, cuda_stream);
			std::vector<uint32_t> segments;
			segments.reserve(entries.size());
			for (const published& entry : entries)
			{
				db->host_tiers[2 * size_t(entry.segment) + t] = entry.metadata;
				segments.push_back(entry.segment);
			}
			if (error == cudaSuccess)
				error = publish(*db, t, segments, cuda_stream);
			if (error != cudaSuccess)
				return check_cuda(context, error, "database_stream_in");
			for (uint32_t chunk = first_chunk; chunk <= last_chunk; ++chunk)
			{
				bit_set(db->loaded[t], chunk, true);
				std::vector<uint32_t>& published_segments = db->chunk_segments[t][chunk];
				for (size_t i = chunk == first_chunk ? 0 : chunk_end[chunk - first_chunk - 1]; i < chunk_end[chunk - first_chunk]; ++i)
					published_segments.push_back(entries[i].segment);
			}
		}
		catch (const std::exception&)
		{
			return set_error(context, ACLB200_ERR_OUT_OF_MEMORY, "database_stream_in: out of host memory");
		}
		if (out_num_chunks != nullptr)
			*out_num_chunks = count;
		return ACLB200_OK;
	}

	aclb200_status aclb200_database_stream_out(aclb200_context* context, aclb200_database* db, uint32_t tier, uint32_t num_chunks,
		uint32_t* out_num_chunks, void* stream)
	{
		aclb200_status status = check_tier(context, db, tier, "database_stream_out");
		if (status != ACLB200_OK)
			return status;
		if (out_num_chunks != nullptr)
			*out_num_chunks = 0;
		const uint32_t t = tier - 1;

		// database.impl.h:548-578: from the first loaded chunk, at most num_chunks
		const uint32_t tier_chunks = db->info.num_chunks[t];
		num_chunks = std::min(num_chunks, tier_chunks);
		uint32_t first_chunk = ~0u;
		for (size_t entry = 0; entry < db->loaded[t].size(); ++entry)
		{
			const uint32_t word = db->loaded[t][entry];
			if (word != 0)
			{
				first_chunk = uint32_t(entry) * 32 + uint32_t(__builtin_clz(word));
				break;
			}
		}
		if (first_chunk == ~0u)
			return ACLB200_OK;
		const uint64_t last64 = uint64_t(first_chunk) + uint64_t(num_chunks) - 1;
		const uint32_t last_chunk = last64 >= uint64_t(tier_chunks) ? tier_chunks - 1 : uint32_t(last64);
		const uint32_t count = last_chunk - first_chunk + 1;
		if (count == 0 || last_chunk < first_chunk)
			return ACLB200_OK;

		try
		{
			// the segments the chunks published (the reference reads the chunk headers back from its streamed in copy, :609-631)
			std::vector<uint32_t> segments;
			for (uint32_t chunk = first_chunk; chunk <= last_chunk; ++chunk)
			{
				for (uint32_t segment : db->chunk_segments[t][chunk])
				{
					db->host_tiers[2 * size_t(segment) + t] = 0;
					segments.push_back(segment);
				}
				db->chunk_segments[t][chunk].clear();
			}

			const bool release = count == bit_count(db->loaded[t]);
			cudaStream_t cuda_stream = static_cast<cudaStream_t>(stream);
			cudaError_t error = cudaSetDevice(context->device);
			if (error == cudaSuccess)
				error = publish(*db, t, segments, cuda_stream);
			if (error == cudaSuccess && release)
			{
				error = cudaFreeAsync(db->d_bulk[t], cuda_stream);
				db->d_bulk[t] = nullptr;
			}
			for (uint32_t chunk = first_chunk; chunk <= last_chunk; ++chunk)
				bit_set(db->loaded[t], chunk, false);
			if (error != cudaSuccess)
				return check_cuda(context, error, "database_stream_out");
		}
		catch (const std::exception&)
		{
			return set_error(context, ACLB200_ERR_OUT_OF_MEMORY, "database_stream_out: out of host memory");
		}
		if (out_num_chunks != nullptr)
			*out_num_chunks = count;
		return ACLB200_OK;
	}

	aclb200_status aclb200_clipset_bind_database(aclb200_context* context, aclb200_clipset* clipset, const aclb200_database* database,
		uint32_t* out_failed_clip)
	{
		if (context == nullptr || clipset == nullptr)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "clipset_bind_database: null context / clip set");
		if (database != nullptr && database->device != clipset->device)
			return set_error(context, ACLB200_ERR_INVALID_ARGUMENT, "clipset_bind_database: the database lives on another device");
		cudaSetDevice(clipset->device);
		if (database == nullptr)
		{
			cudaDeviceSynchronize();
			cudaFree(clipset->d_db_first_segment);
			clipset->d_db_first_segment = nullptr;
			clipset->database = nullptr;
			return ACLB200_OK;
		}

		// decompress.impl.h:105-107 (database_context::contains, database.impl.h:369-405): the clip's runtime clip header must be one the
		// database holds, for a clip of the same hash; its segment headers are then the clip's own
		const uint32_t num_clips = clipset->info.num_clips;
		std::vector<uint32_t> first_segment(num_clips, 0xFFFFFFFFu);
		try
		{
			for (uint32_t clip = 0; clip < num_clips; ++clip)
			{
				const uint32_t offset = clipset->host_blob_db_offset[clip];
				if (offset == 0xFFFFFFFFu)
					continue;
				uint32_t found = 0xFFFFFFFFu;
				for (uint32_t i = 0; i < database->info.num_clips && found == 0xFFFFFFFFu; ++i)
					if (database->clip_header_offset[i] == offset && database->clip_hash[i] == clipset->host_clips[clip].hash)
						found = i;
				const char* why = nullptr;
				if (found == 0xFFFFFFFFu)
					why = "the database does not contain the clip";
				else if (database->clip_num_segments[found] != clipset->host_clips[clip].num_segments)
					why = "the database holds another number of segments for the clip";
				else
				{
					// key frame reads must stay inside the tier buffers: every segment's samples, with the clip's pose size
					const std::vector<uint32_t>& pose_bits = clipset->host_db_pose_bits[clip];
					for (uint32_t s = 0; s < pose_bits.size() && why == nullptr; ++s)
					{
						const uint32_t segment = database->clip_first_segment[found] + s;
						const uint32_t known = database->segment_pose_bits[segment];
						if (known != 0 && known != pose_bits[s])
							why = "another clip set bound the database with other segment sizes";
						for (uint32_t t = 0; t < 2 && why == nullptr; ++t)
						{
							const uint64_t metadata = database->host_tiers[2 * size_t(segment) + t];
							if (metadata != 0 && (metadata >> 32) + (uint64_t(pose_bits[s]) * uint32_t(__builtin_popcount(uint32_t(metadata))) + 7) / 8 > database->info.bulk_data_size[t])
								why = "streamed in samples of the clip lie outside the tier";
						}
					}
				}
				if (why != nullptr)
				{
					if (out_failed_clip != nullptr)
						*out_failed_clip = clip;
					return set_error(context, ACLB200_ERR_INVALID_CLIP, "clipset_bind_database: clip " + std::to_string(clip) + ": " + why);
				}
				first_segment[clip] = database->clip_first_segment[found];
			}
			for (uint32_t clip = 0; clip < num_clips; ++clip)
				if (first_segment[clip] != 0xFFFFFFFFu)
					for (uint32_t s = 0; s < clipset->host_db_pose_bits[clip].size(); ++s)
						database->segment_pose_bits[first_segment[clip] + s] = clipset->host_db_pose_bits[clip][s];
		}
		catch (const std::exception&)
		{
			return set_error(context, ACLB200_ERR_OUT_OF_MEMORY, "clipset_bind_database: out of host memory");
		}

		cudaError_t error = cudaSuccess;
		if (clipset->d_db_first_segment == nullptr)
			error = cudaMalloc(reinterpret_cast<void**>(&clipset->d_db_first_segment), sizeof(uint32_t) * size_t(num_clips));
		else
			error = cudaDeviceSynchronize();		// launches may still read the previous table
		if (error == cudaSuccess)
			error = cudaMemcpy(clipset->d_db_first_segment, first_segment.data(), sizeof(uint32_t) * size_t(num_clips), cudaMemcpyHostToDevice);
		if (error != cudaSuccess)
			return check_cuda(context, error, "clipset_bind_database");
		clipset->database = database;
		return ACLB200_OK;
	}
}
