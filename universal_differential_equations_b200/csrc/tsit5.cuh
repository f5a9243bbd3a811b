// tsit5.cuh -- Tsitouras 5(4) tableau and free 4th-order interpolant as compile-time
// constants (fold into FFMA immediates once the stage loops are unrolled).
//
// Replaces OrdinaryDiffEq's Tsit5ConstantCache used by the reference at
// FisherKPP/Fisher-KPP-CNN.jl:66,132,136, SEIR_exposure/seir_exposure.jl:66,132,
// LotkaVolterra/scenario_1.jl:191.  Values: Tsitouras (2011); they are checked
// against the copy OrdinaryDiffEq serialized into the reference's
// Scenario_1_recovery_0.005.jld2 through the oracle (tests/test_oracle_golden.py)
// and the GPU parity tests.
#pragma once

namespace b200ude {

struct Tsit5 {
    static constexpr int S = 7;
    // c_i (0-based stage index)
    __host__ __device__ static constexpr double c(int i)
    {
        return i == 0 ? 0.0 : i == 1 ? 0.161 : i == 2 ? 0.327 : i == 3 ? 0.9
             : i == 4 ? 0.9800255409045097 : 1.0;
    }
    // a_ij, 0-based, j < i; row 6 is b (FSAL)
    __host__ __device__ static constexpr double a(int i, int j)
    {
        switch (i * 8 + j) {
        case 1 * 8 + 0: return 0.161;
        case 2 * 8 + 0: return -0.008480655492356989;
        case 2 * 8 + 1: return 0.335480655492357;
        case 3 * 8 + 0: return 2.8971530571054935;
        case 3 * 8 + 1: return -6.359448489975075;
        case 3 * 8 + 2: return 4.3622954328695815;
        case 4 * 8 + 0: return 5.325864828439257;
        case 4 * 8 + 1: return -11.748883564062828;
        case 4 * 8 + 2: return 7.4955393428898365;
        case 4 * 8 + 3: return -0.09249506636175525;
        case 5 * 8 + 0: return 5.86145544294642;
        case 5 * 8 + 1: return -12.92096931784711;
        case 5 * 8 + 2: return 8.159367898576159;
        case 5 * 8 + 3: return -0.071584973281401;
        case 5 * 8 + 4: return -0.028269050394068383;
        case 6 * 8 + 0: return 0.09646076681806523;
        case 6 * 8 + 1: return 0.01;
        case 6 * 8 + 2: return 0.4798896504144996;
        case 6 * 8 + 3: return 1.379008574103742;
        case 6 * 8 + 4: return -3.290069515436081;
        case 6 * 8 + 5: return 2.324710524099774;
        default: return 0.0;
        }
    }
    __host__ __device__ static constexpr double b(int j) { return a(6, j); }
    // error weights b_j - btilde_j: err = dt * sum_j bt(j) k_j over the 7 stages
    __host__ __device__ static constexpr double bt(int j)
    {
        switch (j) {
        case 0: return -0.001780011052225777;
        case 1: return -0.0008164344596567469;
        case 2: return 0.007880878010261995;
        case 3: return -0.1447110071732629;
        case 4: return 0.5823571654525552;
        case 5: return -0.45808210592918697;
        case 6: return 0.015151515151515152;
        default: return 0.0;
        }
    }
    // interpolant polynomial coefficients r_{j,p}: b_j(Th) = sum_p r(j,p) Th^p, p = 1..4
    __host__ __device__ static constexpr double r(int j, int p)
    {
        switch (j * 8 + p) {
        case 0 * 8 + 1: return 1.0;
        case 0 * 8 + 2: return -2.763706197274826;
        case 0 * 8 + 3: return 2.9132554618219126;
        case 0 * 8 + 4: return -1.0530884977290216;
        case 1 * 8 + 2: return 0.13169999999999998;
        case 1 * 8 + 3: return -0.2234;
        case 1 * 8 + 4: return 0.1017;
        case 2 * 8 + 2: return 3.9302962368947516;
        case 2 * 8 + 3: return -5.941033872131505;
        case 2 * 8 + 4: return 2.490627285651253;
        case 3 * 8 + 2: return -12.411077166933676;
        case 3 * 8 + 3: return 30.33818863028232;
        case 3 * 8 + 4: return -16.548102889244902;
        case 4 * 8 + 2: return 37.50931341651104;
        case 4 * 8 + 3: return -88.1789048947664;
        case 4 * 8 + 4: return 47.37952196281928;
        case 5 * 8 + 2: return -27.896526289197286;
        case 5 * 8 + 3: return 65.09189467479366;
        case 5 * 8 + 4: return -34.87065786149661;
        case 6 * 8 + 2: return 1.5;
        case 6 * 8 + 3: return -4.0;
        case 6 * 8 + 4: return 2.5;
        default: return 0.0;
        }
    }
    // b_j(Theta)
    __host__ __device__ static constexpr double bTheta(int j, double Th)
    {
        return Th * (r(j, 1) + Th * (r(j, 2) + Th * (r(j, 3) + Th * r(j, 4))));
    }
    // weight of forward stage derivative k_j in u(t_{n+1} - c_i dt), the state the
    // backward (adjoint) stage i needs:  Theta_i = 1 - c_i
    __host__ __device__ static constexpr double bw(int i, int j) { return bTheta(j, 1.0 - c(i)); }
    // b_j(Th) for a run-time Th, in the kernel's precision
    template <typename R>
    __device__ static __forceinline__ void weights(R Th, R (&w)[7])
    {
        w[0] = Th * ((R)r(0, 1) + Th * ((R)r(0, 2) + Th * ((R)r(0, 3) + Th * (R)r(0, 4))));
#pragma unroll
        for (int j = 1; j < 7; ++j) w[j] = Th * Th * ((R)r(j, 2) + Th * ((R)r(j, 3) + Th * (R)r(j, 4)));
    }
};

// The fp32 kernels take (float)bt(j): each weight must round to the same float through double as from its decimal.
static_assert((float)Tsit5::bt(0) == -0.001780011052225777f && (float)Tsit5::bt(1) == -0.0008164344596567469f &&
                  (float)Tsit5::bt(2) == 0.007880878010261995f && (float)Tsit5::bt(3) == -0.1447110071732629f &&
                  (float)Tsit5::bt(4) == 0.5823571654525552f && (float)Tsit5::bt(5) == -0.45808210592918697f &&
                  (float)Tsit5::bt(6) == 0.015151515151515152f,
              "Tsit5 error weights double-round in fp32");

}  // namespace b200ude
