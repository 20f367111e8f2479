// The base pose cache's bookkeeping (acl_b200/csrc/base_pose_cache.h) under the interleavings that host threads sharing one clip set
// can produce. A thread's acquire_base_poses (pipeline.cu) is a hit, or a miss that evicts and inserts; its release_base_poses_use
// unpins after the launch is enqueued. The threads here are named steps: the bookkeeping runs under the clip set's mutex, so a
// sequence of steps is exactly what two threads can produce. The rows are the variant's number.
// Prints PASS and returns 0 when every check holds.
#include "base_pose_cache.h"

#include <stdio.h>

namespace
{
	using Cache = aclb200::BasePoseCache<int>;

	int g_failures = 0;

#define CHECK(cond) do { if (!(cond)) { ++g_failures; printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); } } while (0)

	aclb200::BasePoseKey key_of(int variant)
	{
		aclb200::BasePoseKey key;
		std::memset(&key, 0, sizeof(key));
		key.layout = 48;
		key.default_mode[0] = key.default_mode[1] = 1;
		key.default_mode[2] = 3;
		key.constant_defaults[3] = float(variant);
		return key;
	}

	// acquire_base_poses: the variant's rows, pinned; *evicted = the variant whose rows a miss freed, -1 when none
	bool acquire(Cache& cache, int variant, int* evicted = nullptr)
	{
		if (evicted != nullptr)
			*evicted = -1;
		if (Cache::Entry* hit = cache.acquire(key_of(variant)))
		{
			CHECK(hit->rows == variant);
			return true;
		}
		int gone = -1;
		if (cache.evict(gone) && evicted != nullptr)
			*evicted = gone;
		cache.insert(key_of(variant), variant);
		return false;
	}

	void release(Cache& cache, int variant)
	{
		const int* rows = cache.release(key_of(variant));
		CHECK(rows != nullptr && *rows == variant);
	}

	// pins of the variant, -1 when it is not cached
	int users(Cache& cache, int variant)
	{
		const Cache::Entry* entry = cache.find(key_of(variant));
		return entry == nullptr ? -1 : int(entry->users);
	}

	// the cache holds `count` variants first, first + 1, ..., built and released in that order (oldest first)
	void fill(Cache& cache, int first, int count)
	{
		for (int v = first; v < first + count; ++v)
		{
			CHECK(!acquire(cache, v));
			release(cache, v);
		}
	}

	// Thread A hits X and is setting up its launch; thread B misses on a full cache whose other entries are pinned by launches being
	// set up on other threads. X is pinned too, so B must not free it under A: the cache grows past the cap.
	void hit_pins_against_a_miss_on_a_full_cache(size_t cap)
	{
		Cache cache;
		cache.max_cached = cap;
		const int x = 0;
		fill(cache, x, int(cap));
		for (int v = 1; v < int(cap); ++v)
			CHECK(acquire(cache, v));					// other threads, between their acquire and release
		int evicted = -1;
		CHECK(acquire(cache, x));						// A: hit
		CHECK(users(cache, x) == 1);
		CHECK(!acquire(cache, 100, &evicted));			// B: miss on a full cache
		CHECK(evicted == -1);
		CHECK(users(cache, x) == 1);
		CHECK(cache.entries.size() == cap + 1);
		release(cache, x);								// A has enqueued its launch
		release(cache, 100);
		CHECK(users(cache, x) == 0);
		// X is the least recently used unpinned entry now: the next miss takes it
		CHECK(!acquire(cache, 101, &evicted));
		CHECK(evicted == x);
		CHECK(users(cache, x) == -1);
	}

	// Thread A misses and builds X; thread B hits X and releases it; thread C misses on a full cache. A has not launched yet, so its
	// pin must still hold X.
	void build_stays_pinned_after_another_hit_releases(size_t cap)
	{
		Cache cache;
		cache.max_cached = cap;
		const int x = 0;
		fill(cache, 1, int(cap) - 1);
		for (int v = 1; v < int(cap); ++v)
			CHECK(acquire(cache, v));
		int evicted = -1;
		CHECK(!acquire(cache, x, &evicted));			// A: miss, builds X
		CHECK(evicted == -1);
		CHECK(users(cache, x) == 1);
		CHECK(acquire(cache, x));						// B: hit
		CHECK(users(cache, x) == 2);
		release(cache, x);								// B has enqueued its launch
		CHECK(users(cache, x) == 1);
		CHECK(!acquire(cache, 100, &evicted));			// C: miss on a full cache
		CHECK(evicted == -1);
		CHECK(users(cache, x) == 1);
		CHECK(cache.entries.size() == cap + 1);
		release(cache, x);								// A
		release(cache, 100);
		CHECK(!acquire(cache, 101, &evicted));
		CHECK(evicted == x);
	}

	// Every acquire that returned rows takes one pin, every release gives one back; a release without a pin leaves the count at 0
	void pins_count_acquires()
	{
		Cache cache;
		CHECK(!acquire(cache, 7));
		CHECK(acquire(cache, 7));
		CHECK(acquire(cache, 7));
		CHECK(users(cache, 7) == 3);
		for (int expected = 2; expected >= 0; --expected)
		{
			release(cache, 7);
			CHECK(users(cache, 7) == expected);
		}
		release(cache, 7);
		CHECK(users(cache, 7) == 0);
		CHECK(cache.release(key_of(8)) == nullptr);
	}

	// Every entry pinned: misses grow the cache past the cap. Once unpinned, misses evict again, least recently used first, skipping
	// entries that are pinned; the cache keeps the size it grew to.
	void grows_when_all_pinned_then_evicts_in_lru_order()
	{
		Cache cache;
		cache.max_cached = 4;
		for (int v = 0; v < 6; ++v)
		{
			int evicted = 0;
			CHECK(!acquire(cache, v, &evicted));
			CHECK(evicted == -1);
			CHECK(cache.entries.size() == size_t(v) + 1);
		}
		for (int v : { 2, 0, 5, 1, 3, 4 })
			release(cache, v);
		CHECK(acquire(cache, 0));						// 0 becomes the most recently used
		release(cache, 0);
		CHECK(acquire(cache, 3));						// 3 stays pinned through the misses below
		const int lru_order[] = { 1, 2, 4, 5, 0, 10, 11 };
		for (int i = 0; i < 7; ++i)
		{
			int evicted = -1;
			CHECK(!acquire(cache, 10 + i, &evicted));
			CHECK(evicted == lru_order[i]);
			CHECK(cache.entries.size() == 6);
			release(cache, 10 + i);
		}
		CHECK(users(cache, 3) == 1);
		release(cache, 3);
		int evicted = -1;
		CHECK(!acquire(cache, 20, &evicted));
		CHECK(evicted == 3);
	}

	// Keys that differ in any one field are different variants
	void every_key_field_tells_variants_apart()
	{
		Cache cache;
		cache.max_cached = 64;
		std::vector<aclb200::BasePoseKey> keys(1, key_of(0));
		aclb200::BasePoseKey k = key_of(0);
		k.layout = 40;
		keys.push_back(k);
		k = key_of(0);
		k.normalize_always = 1;
		keys.push_back(k);
		for (int kind = 0; kind < 3; ++kind)
		{
			k = key_of(0);
			k.default_mode[kind] = 2;
			keys.push_back(k);
		}
		for (int i = 0; i < 12; ++i)
		{
			k = key_of(0);
			k.constant_defaults[i] += 0.5f;
			keys.push_back(k);
		}
		for (size_t i = 0; i < keys.size(); ++i)
		{
			CHECK(cache.acquire(keys[i]) == nullptr);
			int evicted = -1;
			CHECK(!cache.evict(evicted));
			cache.insert(keys[i], int(i));
		}
		for (size_t i = 0; i < keys.size(); ++i)
		{
			const Cache::Entry* hit = cache.acquire(keys[i]);
			CHECK(hit != nullptr && hit->rows == int(i));
		}
	}
}

int main()
{
	for (size_t cap : { size_t(1), size_t(4) })
	{
		hit_pins_against_a_miss_on_a_full_cache(cap);
		build_stays_pinned_after_another_hit_releases(cap);
	}
	pins_count_acquires();
	grows_when_all_pinned_then_evicts_in_lru_order();
	every_key_field_tells_variants_apart();
	if (g_failures != 0)
	{
		printf("%d checks failed\n", g_failures);
		return 1;
	}
	printf("PASS\n");
	return 0;
}
