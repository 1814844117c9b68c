// Stand-alone check + timing of the cell-list ball query draft (ball_cells_kernel.cu) on a GPU:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -I pvn3d_b200/csrc -I include \
//        tools/experiments/ball_cells_test.cu pvn3d_b200/csrc/runtime.cu -o tools/experiments/ball_cells_test
// Scene: a raster-ordered depth image of a plane with boxes on it (like the bench clouds), level-1 geometry
// (N = 12288, M = 2048 centres taken from the cloud, radii 0.0175 / 0.025, nsample 16 / 32).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "ball_cells_kernel.cu"

using namespace pvn3d::experiment;

static void cpu_ball_query(const float *cen, const float *xyz, int n, int m, float radius, int ns, int *out) {
  const float r2 = radius * radius;
  for (int j = 0; j < m; ++j) {
    int cnt = 0;
    for (int s = 0; s < ns; ++s) out[j * ns + s] = 0;
    for (int k = 0; k < n && cnt < ns; ++k) {
      const float dx = cen[j * 3] - xyz[k * 3], dy = cen[j * 3 + 1] - xyz[k * 3 + 1], dz = cen[j * 3 + 2] - xyz[k * 3 + 2];
      const float d2 = fmaf(dz, dz, fmaf(dx, dx, dy * dy));
      if (d2 < r2) {
        if (cnt == 0)
          for (int s = 0; s < ns; ++s) out[j * ns + s] = k;
        out[j * ns + cnt] = k;
        ++cnt;
      }
    }
  }
}

int main() {
  const int B = 32, N = 12288, M = 2048, BCHK = 2;
  const float radii[2] = {0.0175f, 0.025f};
  const int ns[2] = {16, 32};
  std::vector<float> xyz(static_cast<size_t>(B) * N * 3), cen(static_cast<size_t>(B) * M * 3);
  srand(7);
  for (int b = 0; b < B; ++b) {
    // 12288 pixels of a 480x640 image in raster order; depth: plane at 1 m with two boxes at 0.7 / 0.8 m
    std::vector<int> pix(N);
    for (int k = 0; k < N; ++k) pix[k] = static_cast<int>((static_cast<long long>(k) * 307200) / N) + rand() % 20;
    for (int k = 0; k < N; ++k) {
      const int row = pix[k] / 640, col = pix[k] % 640;
      float z = 1.0f + 0.0005f * (rand() % 100);
      if (row > 150 && row < 330 && col > 200 && col < 420) z = 0.7f + 0.0005f * (rand() % 100);
      if (row > 60 && row < 140 && col > 450 && col < 600) z = 0.8f + 0.0005f * (rand() % 100);
      float *p = &xyz[(static_cast<size_t>(b) * N + k) * 3];
      p[0] = (col - 320) * z / 572.f;
      p[1] = (row - 240) * z / 572.f;
      p[2] = z;
    }
    for (int j = 0; j < M; ++j) {
      const int k = rand() % N;
      for (int d = 0; d < 3; ++d) cen[(static_cast<size_t>(b) * M + j) * 3 + d] = xyz[(static_cast<size_t>(b) * N + k) * 3 + d];
    }
  }
  CellArgs a{};
  float *d_xyz, *d_cen;
  cudaMalloc(&d_xyz, xyz.size() * 4); cudaMalloc(&d_cen, cen.size() * 4);
  cudaMemcpy(d_xyz, xyz.data(), xyz.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(d_cen, cen.data(), cen.size() * 4, cudaMemcpyHostToDevice);
  a.xyz = d_xyz; a.new_xyz = d_cen; a.n = N; a.m = M; a.cell = 1.001f * radii[1];
  cudaMalloc(&a.sorted, static_cast<size_t>(B) * N * sizeof(float4));
  cudaMalloc(&a.start, static_cast<size_t>(B) * (kCellBuckets + 1) * sizeof(int));
  cudaMalloc(&a.lo, B * 3 * sizeof(float));
  cudaMalloc(&a.overflow, static_cast<size_t>(B) * M);
  for (int r = 0; r < 2; ++r) {
    a.r2[r] = radii[r] * radii[r];
    a.ns[r] = ns[r];
    cudaMalloc(&a.idx[r], static_cast<size_t>(B) * M * ns[r] * sizeof(int));
  }
  cudaEvent_t e0, e1, e2;
  cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventCreate(&e2);
  for (int rep = 0; rep < 3; ++rep) {
    cudaEventRecord(e0);
    cells_build_kernel<<<B, 1024>>>(a);
    cudaEventRecord(e1);
    ball_cells_kernel<<<dim3((M + kCellWarps - 1) / kCellWarps, B), kCellWarps * 32>>>(a);
    cudaEventRecord(e2);
    cudaEventSynchronize(e2);
  }
  float t_build, t_query;
  cudaEventElapsedTime(&t_build, e0, e1);
  cudaEventElapsedTime(&t_query, e1, e2);
  printf("cuda status: %s\n", cudaGetErrorString(cudaGetLastError()));
  printf("B=%d N=%d M=%d: cells_build %.1f us, ball_cells %.1f us\n", B, N, M,
         t_build * 1e3, t_query * 1e3);
  std::vector<unsigned char> over(static_cast<size_t>(B) * M);
  cudaMemcpy(over.data(), a.overflow, over.size(), cudaMemcpyDeviceToHost);
  long n_over = 0;
  for (unsigned char o : over) n_over += o;
  printf("centres left to the index-order scan (more than %d hits): %ld of %d\n", kCellListCap, n_over, B * M);
  long bad = 0, checked = 0;
  for (int r = 0; r < 2; ++r) {
    std::vector<int> got(static_cast<size_t>(B) * M * ns[r]), want(static_cast<size_t>(M) * ns[r]);
    cudaMemcpy(got.data(), a.idx[r], got.size() * sizeof(int), cudaMemcpyDeviceToHost);
    for (int b = 0; b < BCHK; ++b) {
      cpu_ball_query(&cen[static_cast<size_t>(b) * M * 3], &xyz[static_cast<size_t>(b) * N * 3], N, M, radii[r], ns[r], want.data());
      for (int j = 0; j < M; ++j) {
        if (over[static_cast<size_t>(b) * M + j]) continue;
        for (int s = 0; s < ns[r]; ++s, ++checked)
          if (got[(static_cast<size_t>(b) * M + j) * ns[r] + s] != want[j * ns[r] + s]) ++bad;
      }
    }
  }
  printf("index mismatches vs the CPU restatement: %ld of %ld checked\n", bad, checked);
  return bad ? 1 : 0;
}
