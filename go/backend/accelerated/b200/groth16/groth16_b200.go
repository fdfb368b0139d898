//go:build b200

package groth16

import (
	"fmt"

	"github.com/consensys/gnark-crypto/ecc"
	"github.com/consensys/gnark/backend/groth16"
	groth16_bls12377 "github.com/consensys/gnark/backend/groth16/bls12-377"
	groth16_bls12381 "github.com/consensys/gnark/backend/groth16/bls12-381"
	groth16_bn254 "github.com/consensys/gnark/backend/groth16/bn254"
	groth16_bw6761 "github.com/consensys/gnark/backend/groth16/bw6-761"
	"github.com/consensys/gnark/backend/witness"
	"github.com/consensys/gnark/constraint"
	cs_bls12377 "github.com/consensys/gnark/constraint/bls12-377"
	cs_bls12381 "github.com/consensys/gnark/constraint/bls12-381"
	cs_bn254 "github.com/consensys/gnark/constraint/bn254"
	cs_bw6761 "github.com/consensys/gnark/constraint/bw6-761"

	b200_bls12377 "github.com/consensys/gnark/backend/accelerated/b200/groth16/bls12-377"
	b200_bls12381 "github.com/consensys/gnark/backend/accelerated/b200/groth16/bls12-381"
	b200_bn254 "github.com/consensys/gnark/backend/accelerated/b200/groth16/bn254"
	b200_bw6761 "github.com/consensys/gnark/backend/accelerated/b200/groth16/bw6-761"

	"github.com/consensys/gnark/backend/accelerated/b200"
	"github.com/consensys/gnark/backend/accelerated/b200/internal/cabi"
)

// Prove generates the proof of knowledge of a r1cs with full witness (secret + public part).
//
// NB! the provided proving key must be a B200 proving key. Initialize and deserialize the proving key using
// [NewProvingKey] and the serialization methods.
func Prove(r1cs constraint.ConstraintSystem, pk groth16.ProvingKey, fullWitness witness.Witness, opts ...b200.Option) (groth16.Proof, error) {
	config, err := b200.NewConfig(opts...)
	if err != nil {
		return nil, fmt.Errorf("initializing config: %w", err)
	}
	// the twin of warmUpDevice (groth16_icicle.go:38-72): streams and memory pools of the devices, once per process
	if err := cabi.Init(config.Devices()); err != nil {
		panic(fmt.Sprintf("b200 device initialisation: %v", err))
	}
	switch _r1cs := r1cs.(type) {
	case *cs_bls12377.R1CS:
		return b200_bls12377.Prove(_r1cs, pk.(*b200_bls12377.ProvingKey), fullWitness, config)
	case *cs_bls12381.R1CS:
		return b200_bls12381.Prove(_r1cs, pk.(*b200_bls12381.ProvingKey), fullWitness, config)
	case *cs_bn254.R1CS:
		return b200_bn254.Prove(_r1cs, pk.(*b200_bn254.ProvingKey), fullWitness, config)
	case *cs_bw6761.R1CS:
		return b200_bw6761.Prove(_r1cs, pk.(*b200_bw6761.ProvingKey), fullWitness, config)
	default:
		panic("b200 backend requested but r1cs is not of a supported curve")
	}
}

// ProveBatch generates one proof per full witness of one r1cs in a single device call: the witnesses are solved
// concurrently, then every proof's device work runs as one batch (batched NTTs and one batched MSM per key table), which
// pays the fixed cost of the MSM and NTT pipelines once for all of them.  Proof i is what Prove would give for witness i
// with the same randomness.  One device only: WithDevices with more than one device is an error.
//
// NB! the provided proving key must be a B200 proving key.
func ProveBatch(r1cs constraint.ConstraintSystem, pk groth16.ProvingKey, fullWitnesses []witness.Witness, opts ...b200.Option) ([]groth16.Proof, error) {
	config, err := b200.NewConfig(opts...)
	if err != nil {
		return nil, fmt.Errorf("initializing config: %w", err)
	}
	if err := cabi.Init(config.Devices()); err != nil {
		panic(fmt.Sprintf("b200 device initialisation: %v", err))
	}
	out := make([]groth16.Proof, len(fullWitnesses))
	switch _r1cs := r1cs.(type) {
	case *cs_bls12377.R1CS:
		proofs, err := b200_bls12377.ProveBatch(_r1cs, pk.(*b200_bls12377.ProvingKey), fullWitnesses, config)
		for i, p := range proofs {
			out[i] = p
		}
		return out, err
	case *cs_bls12381.R1CS:
		proofs, err := b200_bls12381.ProveBatch(_r1cs, pk.(*b200_bls12381.ProvingKey), fullWitnesses, config)
		for i, p := range proofs {
			out[i] = p
		}
		return out, err
	case *cs_bn254.R1CS:
		proofs, err := b200_bn254.ProveBatch(_r1cs, pk.(*b200_bn254.ProvingKey), fullWitnesses, config)
		for i, p := range proofs {
			out[i] = p
		}
		return out, err
	case *cs_bw6761.R1CS:
		proofs, err := b200_bw6761.ProveBatch(_r1cs, pk.(*b200_bw6761.ProvingKey), fullWitnesses, config)
		for i, p := range proofs {
			out[i] = p
		}
		return out, err
	default:
		panic("b200 backend requested but r1cs is not of a supported curve")
	}
}

// Setup generates a proving and verifying key for a given r1cs.
//
// The method wraps the [groth16.Setup] method, but the returned proving key is a B200 proving key. To convert the key
// to a standard Groth16 proving key, use the serialization methods.
func Setup(r1cs constraint.ConstraintSystem) (groth16.ProvingKey, groth16.VerifyingKey, error) {
	switch _r1cs := r1cs.(type) {
	case *cs_bls12377.R1CS:
		var pk b200_bls12377.ProvingKey
		var vk groth16_bls12377.VerifyingKey
		if err := groth16_bls12377.Setup(_r1cs, &pk.ProvingKey, &vk); err != nil {
			return nil, nil, err
		}
		return &pk, &vk, nil
	case *cs_bls12381.R1CS:
		var pk b200_bls12381.ProvingKey
		var vk groth16_bls12381.VerifyingKey
		if err := groth16_bls12381.Setup(_r1cs, &pk.ProvingKey, &vk); err != nil {
			return nil, nil, err
		}
		return &pk, &vk, nil
	case *cs_bn254.R1CS:
		var pk b200_bn254.ProvingKey
		var vk groth16_bn254.VerifyingKey
		if err := groth16_bn254.Setup(_r1cs, &pk.ProvingKey, &vk); err != nil {
			return nil, nil, err
		}
		return &pk, &vk, nil
	case *cs_bw6761.R1CS:
		var pk b200_bw6761.ProvingKey
		var vk groth16_bw6761.VerifyingKey
		if err := groth16_bw6761.Setup(_r1cs, &pk.ProvingKey, &vk); err != nil {
			return nil, nil, err
		}
		return &pk, &vk, nil
	default:
		panic("b200 backend requested but r1cs is not of a supported curve")
	}
}

// DummySetup generates a dummy proving key for a given circuit. It doesn't perform the precomputations and thus the
// returned proving key cannot be used to generate proofs. The method is useful for development and testing purposes.
func DummySetup(r1cs constraint.ConstraintSystem) (groth16.ProvingKey, error) {
	switch _r1cs := r1cs.(type) {
	case *cs_bls12377.R1CS:
		var pk b200_bls12377.ProvingKey
		if err := groth16_bls12377.DummySetup(_r1cs, &pk.ProvingKey); err != nil {
			return nil, err
		}
		return &pk, nil
	case *cs_bls12381.R1CS:
		var pk b200_bls12381.ProvingKey
		if err := groth16_bls12381.DummySetup(_r1cs, &pk.ProvingKey); err != nil {
			return nil, err
		}
		return &pk, nil
	case *cs_bn254.R1CS:
		var pk b200_bn254.ProvingKey
		if err := groth16_bn254.DummySetup(_r1cs, &pk.ProvingKey); err != nil {
			return nil, err
		}
		return &pk, nil
	case *cs_bw6761.R1CS:
		var pk b200_bw6761.ProvingKey
		if err := groth16_bw6761.DummySetup(_r1cs, &pk.ProvingKey); err != nil {
			return nil, err
		}
		return &pk, nil
	default:
		panic("b200 backend requested but r1cs is not of a supported curve")
	}
}

// NewProvingKey creates a new empty proving key for deserializing into.
//
// The method is compatible with [groth16.NewProvingKey], but returns a B200 proving key.
func NewProvingKey(curveID ecc.ID) groth16.ProvingKey {
	switch curveID {
	case ecc.BLS12_377:
		return &b200_bls12377.ProvingKey{}
	case ecc.BLS12_381:
		return &b200_bls12381.ProvingKey{}
	case ecc.BN254:
		return &b200_bn254.ProvingKey{}
	case ecc.BW6_761:
		return &b200_bw6761.ProvingKey{}
	default:
		panic("b200 backend requested but curve is not supported")
	}
}
