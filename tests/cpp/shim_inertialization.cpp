// tests/cpp/shim_inertialization.cpp -- acl_b200::batch_decompressor::begin_inertialization and inertialize_poses against the C calls they
// wrap: 50 transitions of 23 bones of fabricated poses captured into slots given in reverse order, then 50 poses decayed with mixed records
// (NO_INERTIALIZATION and an out of range record among them); the records and the poses must be byte-identical.
// usage: shim_inertialization; prints PASS, exits 3 without a CUDA device.
#include "../../include/acl_b200/decompress.h"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

int main()
{
	try
	{
		acl_b200::device_context device(0);
		acl_b200::batch_decompressor batch(device);
		const uint32_t num_transitions = 50, num_tracks = 23;
		const size_t pose_floats = size_t(num_tracks) * 12, record_floats = size_t(num_tracks) * 16;
		std::vector<float> poses(4 * num_transitions * pose_floats);
		for (size_t i = 0; i < poses.size(); ++i)
			poses[i] = std::sin(float(i) * 0.37f);
		std::vector<uint32_t> slots(num_transitions);
		std::vector<aclb200_inertialization> inertializations(num_transitions);
		for (uint32_t j = 0; j < num_transitions; ++j)
		{
			slots[j] = num_transitions - 1 - j;
			inertializations[j] = aclb200_inertialization{ j % 7 == 3 ? ACLB200_NO_INERTIALIZATION : (j % 11 == 5 ? num_transitions : j),
				0.01f * float(j), 0.1f + 0.002f * float(j) };
		}
		const size_t poses_bytes = poses.size() * sizeof(float), set_bytes = num_transitions * pose_floats * sizeof(float);
		const size_t records_bytes = num_transitions * record_floats * sizeof(float);
		uint8_t* d_poses = nullptr;
		float* d_records[2] = { nullptr, nullptr };
		float* d_out[2] = { nullptr, nullptr };
		uint32_t* d_slots = nullptr;
		aclb200_inertialization* d_inertializations = nullptr;
		if (cudaMalloc(&d_poses, poses_bytes) != cudaSuccess || cudaMalloc(&d_records[0], records_bytes) != cudaSuccess
			|| cudaMalloc(&d_records[1], records_bytes) != cudaSuccess || cudaMalloc(&d_out[0], set_bytes) != cudaSuccess
			|| cudaMalloc(&d_out[1], set_bytes) != cudaSuccess || cudaMalloc(&d_slots, num_transitions * sizeof(uint32_t)) != cudaSuccess
			|| cudaMalloc(&d_inertializations, num_transitions * sizeof(aclb200_inertialization)) != cudaSuccess)
			return 1;
		cudaMemcpy(d_poses, poses.data(), poses_bytes, cudaMemcpyHostToDevice);
		cudaMemcpy(d_slots, slots.data(), num_transitions * sizeof(uint32_t), cudaMemcpyHostToDevice);
		cudaMemcpy(d_inertializations, inertializations.data(), num_transitions * sizeof(aclb200_inertialization), cudaMemcpyHostToDevice);
		// the same sentinel in both outputs: the poses neither call writes must match too
		cudaMemset(d_out[0], 0xAB, set_bytes);
		cudaMemset(d_out[1], 0xAB, set_bytes);
		const uint8_t* src = d_poses;
		const uint8_t* src_prev = d_poses + set_bytes;
		const uint8_t* dst = d_poses + 2 * set_bytes;
		const uint8_t* dst_prev = d_poses + 3 * set_bytes;
		batch.begin_inertialization(src, src_prev, dst, dst_prev, num_transitions, num_tracks, 30.0f, d_records[0], d_slots);
		if (aclb200_begin_inertialization(device.get(), src, src_prev, dst, dst_prev, num_transitions, num_tracks, 0, 30.0f, d_records[1], 0, d_slots,
			nullptr) != ACLB200_OK)
			return 1;
		batch.inertialize_poses(dst, d_out[0], num_transitions, num_tracks, d_inertializations, d_records[0], num_transitions);
		if (aclb200_inertialize_poses(device.get(), dst, d_out[1], num_transitions, num_tracks, 0, d_inertializations, d_records[1], num_transitions,
			0, nullptr) != ACLB200_OK)
			return 1;
		std::vector<uint8_t> records[2] = { std::vector<uint8_t>(records_bytes), std::vector<uint8_t>(records_bytes) };
		std::vector<uint8_t> out[2] = { std::vector<uint8_t>(set_bytes), std::vector<uint8_t>(set_bytes) };
		for (int i = 0; i < 2; ++i)
			if (cudaMemcpy(records[i].data(), d_records[i], records_bytes, cudaMemcpyDeviceToHost) != cudaSuccess
				|| cudaMemcpy(out[i].data(), d_out[i], set_bytes, cudaMemcpyDeviceToHost) != cudaSuccess)
				return 1;
		if (std::memcmp(records[0].data(), records[1].data(), records_bytes) != 0 || std::memcmp(out[0].data(), out[1].data(), set_bytes) != 0)
		{
			std::printf("FAIL shim and C call differ\n");
			return 1;
		}
		cudaFree(d_poses);
		cudaFree(d_records[0]);
		cudaFree(d_records[1]);
		cudaFree(d_out[0]);
		cudaFree(d_out[1]);
		cudaFree(d_slots);
		cudaFree(d_inertializations);
	}
	catch (const acl_b200::error& e)
	{
		std::fprintf(stderr, "%s\n", e.what());
		return e.status == ACLB200_ERR_NO_DEVICE ? 3 : 1;
	}
	std::printf("PASS\n");
	return 0;
}
