// Development experiment: how fast can an H100 drain 2.4 GB of pose rows through 1-D TMA bulk stores (cp.async.bulk shared -> global),
// nothing else going on? The floor of the pipeline kernel's output side.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tma_store_floor tma_store_floor.cu && ./tma_store_floor
// Each block owns a contiguous range of the output and loops: (optionally touch the chunk in shared memory) -> fence -> one bulk store
// of `chunk` bytes -> commit; a stage is reused once wait_group.read says the copy has read it.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

template<int STAGES>
__global__ void __launch_bounds__(128) store_kernel(uint8_t* out, uint64_t total_bytes, uint32_t chunk, int touch)
{
	extern __shared__ __align__(128) uint8_t smem[];
	const uint64_t chunks = total_bytes / chunk;
	const uint64_t share = chunks / gridDim.x, rem = chunks % gridDim.x;
	const uint64_t first = blockIdx.x * share + (blockIdx.x < rem ? blockIdx.x : rem);
	const uint64_t count = share + (blockIdx.x < rem ? 1 : 0);
	for (uint64_t i = 0; i < count; ++i)
	{
		uint8_t* stage = smem + (i % STAGES) * chunk;
		if (threadIdx.x == 0 && i >= STAGES)
			asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(STAGES - 1) : "memory");
		__syncthreads();
		if (touch)
			for (uint32_t b = threadIdx.x * 16; b < chunk; b += blockDim.x * 16)
				*reinterpret_cast<float4*>(stage + b) = make_float4(float(i), 1.f, 2.f, 3.f);
		asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
		__syncthreads();
		if (threadIdx.x == 0)
		{
			const uint32_t src = static_cast<uint32_t>(__cvta_generic_to_shared(stage));
			asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" :: "l"(out + (first + i) * chunk), "r"(src), "r"(chunk) : "memory");
			asm volatile("cp.async.bulk.commit_group;" ::: "memory");
		}
	}
	if (threadIdx.x == 0)
		asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

__global__ void plain_store_kernel(float4* out, uint64_t n)
{
	const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
	for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
		out[i] = make_float4(float(i), 1.f, 2.f, 3.f);
}

template<int STAGES>
float run(uint8_t* out, uint64_t total, uint32_t chunk, int blocks_per_sm, int touch)
{
	cudaFuncSetAttribute(store_kernel<STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, STAGES * chunk);
	cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
	float best = 1e9f;
	for (int r = 0; r < 4; ++r)
	{
		cudaEventRecord(a);
		store_kernel<STAGES><<<132 * blocks_per_sm, 128, STAGES * chunk>>>(out, total, chunk, touch);
		cudaEventRecord(b); cudaEventSynchronize(b);
		float ms; cudaEventElapsedTime(&ms, a, b);
		if (r > 0 && ms < best) best = ms;
	}
	return best;
}

int main()
{
	const uint64_t total = 2400000000ull;
	uint8_t* out;
	cudaMalloc(&out, total + (1 << 20));
	cudaMemset(out, 0, total);
	{
		cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
		for (int r = 0; r < 3; ++r)
		{
			cudaEventRecord(a);
			plain_store_kernel<<<132 * 8, 256>>>(reinterpret_cast<float4*>(out), total / 16);
			cudaEventRecord(b); cudaEventSynchronize(b);
			float ms; cudaEventElapsedTime(&ms, a, b);
			if (r == 2) printf("plain coalesced 16 B stores: %.3f ms  %.0f GB/s\n", ms, total / ms / 1e6);
		}
		cudaEventRecord(a);
		cudaMemsetAsync(out, 1, total);
		cudaEventRecord(b); cudaEventSynchronize(b);
		float ms; cudaEventElapsedTime(&ms, a, b);
		printf("cudaMemset: %.3f ms  %.0f GB/s\n", ms, total / ms / 1e6);
	}
	const uint32_t chunks[] = { 40000, 48000, 16000, 8000, 4000 };
	for (uint32_t chunk : chunks)
		for (int bps = 1; bps <= 4; bps *= 2)
			for (int touch = 0; touch <= 1; ++touch)
			{
				if (2 * chunk * bps > 220000) continue;
				const float t2 = run<2>(out, total, chunk, bps, touch);
				const float t1 = run<1>(out, total, chunk, bps, touch);
				printf("chunk %6u B  blocks/SM %d  touch %d :  2 stages %.3f ms (%.0f GB/s)   1 stage %.3f ms (%.0f GB/s)\n", chunk, bps, touch,
					t2, total / t2 / 1e6, t1, total / t1 / 1e6);
			}
	return 0;
}
