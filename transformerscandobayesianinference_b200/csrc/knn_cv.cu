// KNN baseline of the tabular evaluation (reference tabular.py:350-369 knn_metric): per problem
//   GridSearchCV(KNeighborsClassifier(), {'n_neighbors': arange(1, min(6, n - 1))}, cv=min(5, n // 2)).fit(x, y)
//   followed by predict_proba(test_x)[:, 1]
// for ALL problems of a (dataset, eval position) in one launch, one CTA per problem.
//
// The folds are sklearn's StratifiedKFold without shuffling (_make_test_folds): classes encoded by order of first
// appearance, allocation[i, k] = bincount(sort(y_enc)[i::n_splits])[k], and the rows of class k take
// repeat(arange(n_splits), allocation[:, k]) in row order.  Neighbours are uniform-weight Euclidean, ordered by (squared
// distance, train row index), the squared distances summed feature by feature in fp64 from direct differences (no
// contraction into FMAs, so the CPU restatement oracle/tabular_oracle.py reproduces them bit for bit).  A vote tie predicts
// class 0 (sklearn's argmax over the sorted classes).  A fold's accuracy is correct / n_fold in fp64; a candidate's mean is
// the fold accuracies summed left to right over the folds, divided by the fold count (numpy's mean for <= 7 folds).  A
// candidate k larger than a fold's training set scores NaN there (sklearn's error_score) and NaN candidates rank last.
// The best candidate is the first maximal mean (rank_test_score.argmin()); the refit on all n rows gives
// proba = count_1 / k per test row.
#include "common.cuh"
#include "../../include/pfn_b200.h"

namespace pfn {
namespace {

constexpr int kThreads = 256;
constexpr int KMAX = PFN_KNN_MAX_K;

__device__ __forceinline__ double sq_dist(const float* __restrict__ a, const float* __restrict__ b, int F) {
  double d = 0.0;
  for (int f = 0; f < F; ++f) {
    const double t = static_cast<double>(a[f]) - static_cast<double>(b[f]);
    d = __dadd_rn(d, __dmul_rn(t, t));
  }
  return d;
}

// the KMAX nearest rows seen so far, ordered by (distance, row); rows arrive in increasing order, so an equal distance
// goes behind the ones already kept.  Only the neighbours' labels are needed.
struct TopK {
  double d[KMAX];
  int lab[KMAX];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int t = 0; t < KMAX; ++t) { d[t] = INFINITY; lab[t] = 0; }
  }
  __device__ __forceinline__ void push(double dist, int label) {
    if (!(dist < d[KMAX - 1])) return;
    int pos = KMAX - 1;
#pragma unroll
    for (int t = KMAX - 2; t >= 0; --t) if (dist < d[t]) pos = t;
#pragma unroll
    for (int t = KMAX - 1; t > 0; --t) if (t > pos) { d[t] = d[t - 1]; lab[t] = lab[t - 1]; }
#pragma unroll
    for (int t = 0; t < KMAX; ++t) if (t == pos) { d[t] = dist; lab[t] = label; }
  }
  __device__ __forceinline__ int ones(int k) const {
    int c = 0;
#pragma unroll
    for (int t = 0; t < KMAX; ++t) c += (t < k) ? lab[t] : 0;
    return c;
  }
};

// number of j in [0, x) with j % ns == i
__device__ __forceinline__ int residue_count(int x, int ns, int i) { return x / ns + (i < x % ns ? 1 : 0); }

__global__ void __launch_bounds__(kThreads) knn_cv_kernel(pfn_knn_cv_desc D) {
  __shared__ unsigned char lab[PFN_KNN_MAX_N];
  __shared__ unsigned char fold[PFN_KNN_MAX_N];
  __shared__ int correct[PFN_KNN_MAX_SPLITS][KMAX];
  __shared__ int fold_size[PFN_KNN_MAX_SPLITS];
  __shared__ int sh_status, sh_k;

  const int s = blockIdx.x, tid = threadIdx.x;
  const int n = D.n, m = D.m, F = D.F, S = D.S;
  const int ns = n / 2 < 5 ? n / 2 : 5;
  const int K = n - 2 < KMAX ? n - 2 : KMAX;
  const size_t row_stride = static_cast<size_t>(S) * F;
  const float* xs = D.x + static_cast<size_t>(s) * F;

  for (int t = tid; t < PFN_KNN_MAX_SPLITS * KMAX; t += kThreads) correct[t / KMAX][t % KMAX] = 0;
  if (tid == 0) {
    int status = PFN_KNN_OK;
    for (int r = 0; r < n; ++r) {
      const float v = D.y[static_cast<size_t>(r) * S + s];
      if (!(v == 0.0f || v == 1.0f)) status = PFN_KNN_BAD_LABEL;
      lab[r] = v == 1.0f ? 1 : 0;
    }
    if (status == PFN_KNN_OK) {
      // encoded class 0 is the label of row 0 (order of first appearance)
      int count[2] = {0, 0};
      for (int r = 0; r < n; ++r) ++count[lab[r] != lab[0]];
      if (count[1] == 0) status = PFN_KNN_ONE_CLASS;
      else if (ns > count[0] && ns > count[1]) status = PFN_KNN_FEW_MEMBERS;
      if (status == PFN_KNN_OK) {
        // allocation[i][k] over sort(y_enc) = [0] * count[0] + [1] * count[1]
        int alloc[PFN_KNN_MAX_SPLITS][2];
        for (int i = 0; i < ns; ++i) {
          alloc[i][0] = residue_count(count[0], ns, i);
          alloc[i][1] = residue_count(n, ns, i) - alloc[i][0];
          fold_size[i] = alloc[i][0] + alloc[i][1];
        }
        int f_of[2] = {0, 0}, used[2] = {0, 0};
        for (int r = 0; r < n; ++r) {
          const int k = lab[r] != lab[0];
          while (used[k] == alloc[f_of[k]][k]) { ++f_of[k]; used[k] = 0; }
          fold[r] = static_cast<unsigned char>(f_of[k]);
          ++used[k];
        }
      }
    }
    sh_status = status;
    D.status[s] = status;
  }
  __syncthreads();
  if (sh_status != PFN_KNN_OK) {
    for (int k = tid; k < K; k += kThreads) D.cv_mean[static_cast<size_t>(s) * K + k] = NAN;
    for (int r = tid; r < m; r += kThreads) D.proba[static_cast<size_t>(r) * S + s] = NAN;
    if (tid == 0) D.k_best[s] = 0;
    return;
  }

  // cross-validation: every train row is a query of its own test fold against the other folds' rows
  for (int i = tid; i < n; i += kThreads) {
    const float* xi = xs + i * row_stride;
    const int fi = fold[i];
    TopK best;
    best.init();
    for (int j = 0; j < n; ++j)
      if (fold[j] != fi) best.push(sq_dist(xi, xs + j * row_stride, F), lab[j]);
    const int avail = n - fold_size[fi];
    for (int k = 1; k <= K && k <= avail; ++k) {
      const int c1 = best.ones(k);
      const int pred = 2 * c1 > k ? 1 : 0;
      if (pred == lab[i]) atomicAdd(&correct[fi][k - 1], 1);
    }
  }
  __syncthreads();

  if (tid == 0) {
    int kb = 1;
    double best_mean = NAN;
    for (int k = 1; k <= K; ++k) {
      double sum = 0.0;
      bool nan = false;
      for (int f = 0; f < ns; ++f) {
        if (k > n - fold_size[f]) { nan = true; continue; }
        sum += static_cast<double>(correct[f][k - 1]) / static_cast<double>(fold_size[f]);
      }
      const double mean = nan ? NAN : sum / static_cast<double>(ns);
      D.cv_mean[static_cast<size_t>(s) * K + k - 1] = mean;
      if (!isnan(mean) && (isnan(best_mean) || mean > best_mean)) { best_mean = mean; kb = k; }
    }
    sh_k = kb;
    D.k_best[s] = kb;
  }
  __syncthreads();

  // refit on all n rows with the chosen k
  const int k = sh_k;
  for (int r = tid; r < m; r += kThreads) {
    const float* xr = xs + (n + r) * row_stride;
    TopK best;
    best.init();
    for (int j = 0; j < n; ++j) best.push(sq_dist(xr, xs + j * row_stride, F), lab[j]);
    D.proba[static_cast<size_t>(r) * S + s] = static_cast<double>(best.ones(k)) / static_cast<double>(k);
  }
}

}  // namespace
}  // namespace pfn

extern "C" int pfn_knn_cv(const pfn_knn_cv_desc* d, void* stream) {
  using namespace pfn;
  PFN_CHECK_ARG(d != nullptr, "knn_cv: null descriptor");
  PFN_CHECK_ARG(d->S > 0 && d->m > 0 && d->F > 0, "knn_cv: empty problem S=%d m=%d F=%d", d->S, d->m, d->F);
  PFN_CHECK_ARG(d->n >= 4 && d->n <= PFN_KNN_MAX_N, "knn_cv: n=%d training rows outside [4, %d]", d->n, PFN_KNN_MAX_N);
  PFN_CHECK_ARG(d->F <= PFN_KNN_MAX_F, "knn_cv: F=%d features exceed %d", d->F, PFN_KNN_MAX_F);
  PFN_CHECK_ARG(d->x && d->y && d->proba && d->k_best && d->cv_mean && d->status, "knn_cv: null pointer in the descriptor");
  knn_cv_kernel<<<d->S, kThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(*d);
  PFN_LAUNCH_OK();
  return 0;
}
