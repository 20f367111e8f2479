// acl_b200/csrc/base_pose_cache.h -- the bookkeeping of a clip set's cached base pose rows (pipeline.cu): which variant a launch
// gets, which variants are pinned, which one is evicted. No CUDA calls: pipeline.cu allocates, builds, waits on and frees the rows,
// and tests/cpp/base_pose_cache.cpp replays the interleavings of several host threads on the same bookkeeping.
#pragma once

#include <stddef.h>
#include <stdint.h>
#include <cstring>
#include <vector>

namespace aclb200
{
	// What a clip's base pose row (constant + default sub-tracks in the output layout, pipeline.cu) depends on besides the clip.
	// Compared bytewise: no padding, and whoever fills one clears it first.
	struct BasePoseKey
	{
		uint32_t layout;
		uint32_t normalize_always;
		uint32_t default_mode[3];
		float    constant_defaults[12];
	};

	// The base pose variants of one clip set. Every acquire that returns an entry, hit or miss, pins it until its matching release,
	// so a launch being set up with an entry's rows never sees them evicted. Eviction takes the least recently used unpinned entry
	// once the cache holds max_cached entries; when every entry is pinned the cache grows past max_cached instead. Not locked: the
	// caller holds the clip set's base_mutex around every call and around what it does with the entry it got.
	template<typename Rows>
	struct BasePoseCache
	{
		struct Entry
		{
			BasePoseKey key;
			Rows rows;
			uint32_t users;			// launches being set up with these rows: one per acquire or insert until its release
			uint64_t last_use;
		};

		size_t max_cached = 4;
		std::vector<Entry> entries;
		uint64_t clock = 0;

		// A hit: the entry, pinned and made the most recently used. nullptr on a miss.
		Entry* acquire(const BasePoseKey& key)
		{
			Entry* entry = find(key);
			if (entry != nullptr)
			{
				entry->last_use = ++clock;
				entry->users++;
			}
			return entry;
		}

		// A miss, before it builds its rows: when the cache is full, takes the least recently used unpinned entry out and hands its rows
		// to the caller to free. false when nothing had to go, or when every entry is pinned.
		bool evict(Rows& evicted)
		{
			if (entries.size() < max_cached)
				return false;
			size_t oldest = entries.size();
			for (size_t i = 0; i < entries.size(); ++i)
				if (entries[i].users == 0 && (oldest == entries.size() || entries[i].last_use < entries[oldest].last_use))
					oldest = i;
			if (oldest == entries.size())
				return false;
			evicted = entries[oldest].rows;
			entries.erase(entries.begin() + oldest);
			return true;
		}

		// The rows a miss built: a new entry, pinned by that miss
		void insert(const BasePoseKey& key, const Rows& rows)
		{
			Entry entry;
			entry.key = key;
			entry.rows = rows;
			entry.users = 1;
			entry.last_use = ++clock;
			entries.push_back(entry);
		}

		// Unpins the entry an acquire or insert pinned: its rows, nullptr when no entry has the key
		Rows* release(const BasePoseKey& key)
		{
			Entry* entry = find(key);
			if (entry == nullptr)
				return nullptr;
			if (entry->users != 0)
				entry->users--;
			return &entry->rows;
		}

		Entry* find(const BasePoseKey& key)
		{
			for (Entry& entry : entries)
				if (std::memcmp(&entry.key, &key, sizeof(key)) == 0)
					return &entry;
			return nullptr;
		}
	};
}
